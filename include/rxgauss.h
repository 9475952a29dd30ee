/* rxgauss.h -- C ABI of librxgauss: H100 (sm_90a) kernels for the Gaussian message-passing hot
 * path of RxInfer.jl's infer().
 *
 * This header is the drop-in boundary.  Every entry point replaces one piece of the reference's
 * per-message / per-chain machinery; the reference-side interface each one stands in for is cited
 * as  [ref: file:line]  relative to /root/reference.  Rule bodies marked (upstream) live in the
 * un-vendored ReactiveMP ~6.0.0 / ExponentialFamily 2.1.0 / BayesBase 1.5.0 / FastCholesky 1.3.0
 * (Project.toml:43-73); the in-repo citation is the call site that binds or exercises them.
 *
 * Conventions
 *  - plain C, no exceptions, no callbacks.  Every function returns an rxg_status (0 = OK);
 *    rxg_last_error(ctx) gives a human-readable message for the last failure on that ctx.
 *  - all arrays are fp32, structure-of-arrays with the batch (message / chain) index INNERMOST:
 *        vectors  v[k][n]          -> v[k*n_total + i]
 *        matrices M[r][c][n]       -> M[(r*C + c)*n_total + i]
 *        series   y[t][k][batch]   -> y[(t*m + k)*batch + b]
 *    so that a warp reading one component of 32 consecutive chains issues one 128-byte request.
 *  - (mu, Sigma) = mean / covariance  (MvNormalMeanCovariance),
 *    (xi, W)     = weighted mean / precision (MvNormalWeightedMeanPrecision), W = inv(Sigma), xi = W mu.
 *  - pointers are device pointers when RXG_PTR_DEVICE is set in `flags`, host pointers otherwise
 *    (host buffers are staged through the context's stream; pinned memory from rxg_host_alloc
 *    makes the copies asynchronous).
 *  - the caller owns every buffer it passes; the library owns only what hangs off rxg_ctx
 *    (stream handle, workspace, gain tables, NCCL communicator).
 *  - a ctx is bound to one device and is not thread-safe: one ctx per host thread and per GPU.
 *  - calls return after the stream has been synchronised unless RXG_ASYNC is set.
 *  - there is NO CPU fallback: without a usable CUDA device rxg_create fails with
 *    RXG_ERR_NO_DEVICE and every compute entry point fails with RXG_ERR_BAD_ARG on a null ctx.
 */
#ifndef RXGAUSS_H
#define RXGAUSS_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define RXG_VERSION 100 /* 0.1.0 */

typedef struct rxg_ctx rxg_ctx;

typedef enum rxg_status {
    RXG_OK = 0,
    RXG_ERR_BAD_ARG = 1,
    RXG_ERR_CUDA = 2,
    RXG_ERR_NCCL = 3,
    RXG_ERR_NOT_SPD = 4,     /* at least one chain/message hit a non-positive Cholesky pivot      */
    RXG_ERR_NAN = 5,
    RXG_ERR_UNSUPPORTED = 6, /* shape outside the compiled kernel families (see rxg_supports)   */
    RXG_ERR_NO_DEVICE = 7
} rxg_status;

enum rxg_flags {
    RXG_PTR_DEVICE      = 1u << 0, /* data pointers are device pointers                          */
    RXG_MODEL_PER_CHAIN = 1u << 1, /* A,B,P,Q,m0,S0 carry a trailing [batch] axis               */
    RXG_ASYNC           = 1u << 2, /* do not synchronise the stream before returning             */
    RXG_COV_SHARED_OUT  = 1u << 3, /* shared model only: write post_cov as [T][d][d] (one copy)  */
    RXG_PATH_PER_CHAIN  = 1u << 4, /* force the per-chain covariance recursion (no gain tables)  */
    RXG_TRANSITION_FIRST = 1u << 5, /* the prior sits one transition before the first datum      */
    RXG_COV_REPLICATE   = 1u << 6, /* all-gather: covariances are chain independent (shared model,
                                      no missing data) -- replicate them locally, gather only means */
    RXG_MASK_SHARED     = 1u << 7, /* ymask is ONE pattern for all chains: a HOST array ymask[T] (like the model
                                      matrices).  The covariances stay chain independent, so the call stays on the
                                      gain-table path (a per-chain mask forces the per-chain covariance recursion,
                                      ~2.7x slower at d = 4).  y at masked steps is ignored but must be finite.   */
    /* Known per-step inputs (control / exogenous terms): `u` is a SEQUENCE, x[t] ~ N(A x[t-1] + u[t], P).  Row t
     * (0-based) enters the transition into x[t]; row 0 is read only with RXG_TRANSITION_FIRST.  A masked step still
     * applies its input.  Inputs move only the means: covariances (and gain tables) are those of the call without
     * inputs.  A constant offset has to be folded into the sequence by the caller.  Both flags together: BAD_ARG.  */
    RXG_U_SEQ_SHARED    = 1u << 8, /* u is ONE sequence for every chain: a HOST array u[rows][d] (also with
                                      RXG_MODEL_PER_CHAIN)                                                        */
    RXG_U_SEQ_CHAIN     = 1u << 9  /* u is a DEVICE array u[rows][d][batch] (shared or per-chain model); needs
                                      RXG_PTR_DEVICE (host-pointer calls return RXG_ERR_UNSUPPORTED)              */
};

/* Per-context options (rxg_set_option).  The RXG_* environment variables of the same name are read
 * ONCE, inside rxg_create, as the initial values; nothing on a compute path calls getenv.        */
typedef enum rxg_option {
    RXG_OPT_GAIN_SEQ = 0,          /* 1: sequential Riccati gain kernels (cross-check of the time-parallel scan)   */
    RXG_OPT_LARGE_SEQ = 1,         /* 1: sequential gain kernels of the large-state family (cross-check)            */
    RXG_OPT_NO_UMMA = 2,           /* 1: d >= 16 mean recursions on the FP32 pipe instead of wgmma (cross-check)    */
    RXG_OPT_SWEEP_VARIANT = 3,     /* shared-model sweep: 0 auto, 1 stash, 3 time-segmented (experimental, slower)  */
    RXG_OPT_FORCE_CPT = 4,         /* chains per thread of the shared-model sweep (0 = auto)                        */
    RXG_OPT_HOST_THREADS = 5,      /* host threads of the host-side covariance broadcast (0 = auto)                 */
    RXG_OPT_HOST_COV_D2H = 6,      /* 1: host-pointer calls copy the per-chain covariances over PCIe (no broadcast) */
    RXG_OPT_HOST_BCAST_MIN_MB = 7, /* below this covariance size the host broadcast is not used (default 64)        */
    RXG_OPT_HOST_SLICES = 8,       /* batch slices of the host-pointer pipeline (0 = auto)                          */
    RXG_OPT_GATHER_MODE = 9,       /* rxg_lgssm_smooth_gather_f32: 0/1 peer stores fused into the sweep, 2 push after it  */
    RXG_OPT_POLYA_PATH = 10,       /* rxg_binomial_polya_vmp_f32: 0 auto, 1 one thread per chain, 2 chain groups (cross-check) */
    RXG_OPT_COUNT_ = 11
} rxg_option;

#define RXG_MAX_PEERS 8            /* ranks of one peer group (one NVSwitch domain)                                 */

/* ------------------------------------------------------------------ context / plumbing ------ */
int rxg_version(void);
/* Create a context on CUDA device `device`.  [ref: the reference has no device/ctx notion; this
 * replaces the per-infer() engine state built at src/inference/batch.jl:177-257]               */
int rxg_create(rxg_ctx** out, int device, unsigned flags);
int rxg_destroy(rxg_ctx* ctx);
const char* rxg_last_error(const rxg_ctx* ctx);
int rxg_set_option(rxg_ctx* ctx, int option, long long value);
int rxg_get_option(const rxg_ctx* ctx, int option, long long* value);
/* Use an externally owned cudaStream_t (e.g. torch's current stream) for all launches/copies.  */
int rxg_set_stream(rxg_ctx* ctx, void* cuda_stream);
int rxg_sync(rxg_ctx* ctx);
/* Pinned host memory for asynchronous staging of host-pointer calls.                           */
int rxg_host_alloc(void** out, size_t bytes);
int rxg_host_free(void* p);
/* 1 if the fused sweeps accept (d, m): any 1 <= d, m <= 64.  Shapes without a dedicated kernel family are
 * embedded in the next larger one (shared model) or run on the generic one-CTA-per-chain kernel (per-chain
 * models, missing data); see csrc/rxg_lgssm_general.cu.                                          */
int rxg_supports(int d, int m);
/* Host threads the library will use to broadcast chain-independent covariances into a HOST output
 * buffer (host-pointer calls of a shared model fetch the [T][d][d] table once instead of copying the
 * per-chain duplicates over PCIe): RXG_HOST_THREADS, else min(affinity, cgroup quota, 16) divided by
 * LOCAL_WORLD_SIZE.  Below 6 the full device->host copy is used (also forced by RXG_HOST_COV_D2H=1). */
int rxg_host_fill_threads(void);
/* Number of kernels this ctx has launched so far (for bench.py's gpu_launches).               */
long long rxg_launch_count(const rxg_ctx* ctx);
/* Per-kernel timing of the most recent fused LGSSM sweep: when enabled, CUDA events are recorded
 * on the ctx stream around the gain-table kernels and around the dominant sweep kernel.
 * rxg_profile_last_ms synchronises on those events; *gain_ms is 0 on the per-chain path.        */
int rxg_set_profiling(rxg_ctx* ctx, int enabled);
int rxg_profile_last_ms(rxg_ctx* ctx, float* main_kernel_ms, float* gain_kernels_ms);

/* ------------------------------------------------------------------ per-rule kernels --------
 * Batched twins of the reference's @rule bodies: n independent messages per call, pure
 * functions.  `M_shared != 0` means the PointMass matrix operand is one d x d (row-major) matrix
 * shared by all n messages, else it is [r][c][n].
 * The reference reaches these through ReactiveMP.rule(...) dispatched from the edge pipelines
 * wired in activate_rmp_factornode! [ref: src/model/plugins/reactivemp_inference.jl:509-540];
 * callable directly as @call_rule [ref: test/inference/inference_tests.jl:547-585].
 * State sizes: any 1 <= d <= 64 (d_out, d_in <= 64 for the multiplication rules).  d in {1..6, 8} (and the rectangular
 * shapes 1x2, 1x4, 2x4) run register resident, one thread per message; every other size runs on the shared-memory /
 * left-GEMM kernels of csrc/rxg_rules_large.cu, where the multiplication rules need M_shared != 0.                  */

/* @rule MvNormalMeanCovariance(:out)(m_mu, q_Sigma) -> (mu, S + Sigma)  (upstream
 * rules/mv_normal_mean_covariance/out.jl)  [ref: alias src/model/graphppl.jl:372-376;
 * benchmarks/Linear...Benchmark.ipynb:102]                                                      */
int rxg_rule_mvnormal_meancov_out_f32(rxg_ctx*, int64_t n, int d, const float* mu_in,
                                      const float* S_in, const float* Sigma, int M_shared,
                                      float* mu_out, float* S_out, unsigned flags);
/* @rule MvNormalMeanCovariance(:mu)(m_out, q_Sigma) -> (mu_out, S_out + Sigma)  (upstream
 * .../mean.jl)  [ref: ipynb:102-103]                                                             */
int rxg_rule_mvnormal_meancov_mean_f32(rxg_ctx*, int64_t n, int d, const float* mu_in,
                                       const float* S_in, const float* Sigma, int M_shared,
                                       float* mu_out, float* S_out, unsigned flags);
/* same rule with q_out::PointMass (a datum pushed by new_observation!
 * [ref: src/inference/batch.jl:405-407]) -> (y, Sigma)                                          */
int rxg_rule_mvnormal_meancov_mean_data_f32(rxg_ctx*, int64_t n, int d, const float* y,
                                            const float* Sigma, int M_shared, float* mu_out,
                                            float* S_out, unsigned flags);
/* @rule typeof(*)(:out)(m_A::PointMass, m_in) -> (A mu, A S A')  (upstream
 * rules/multiplication/out.jl)  [ref: ipynb:102; src/model/graphppl.jl:58-83]; A is d_out x d_in */
int rxg_rule_mul_out_f32(rxg_ctx*, int64_t n, int d_out, int d_in, const float* A, int M_shared,
                         const float* mu_in, const float* S_in, float* mu_out, float* S_out,
                         unsigned flags);
/* @rule typeof(*)(:in)(m_out, m_A::PointMass) -> (xi, W) = (A' W_out mu_out, A' W_out A) with
 * W_out = cholinv(S_out)  (upstream rules/multiplication/in.jl).  status[n] (optional) receives
 * RXG_ERR_NOT_SPD per message.                                                                  */
int rxg_rule_mul_in_f32(rxg_ctx*, int64_t n, int d_out, int d_in, const float* A, int M_shared,
                        const float* mu_out, const float* S_out, float* xi_in, float* W_in,
                        int32_t* status, unsigned flags);
/* @rule typeof(+)(:out) -> (mu1 + mu2, S1 + S2); (:in1)/(:in2) -> (mu_out - mu_other, S_out +
 * S_other)  (upstream rules/addition)  [ref: test/models/statespace/ulgssm_tests.jl:12]         */
int rxg_rule_add_out_f32(rxg_ctx*, int64_t n, int d, const float* mu1, const float* S1,
                         const float* mu2, const float* S2, float* mu_out, float* S_out,
                         unsigned flags);
int rxg_rule_add_in_f32(rxg_ctx*, int64_t n, int d, const float* mu_out, const float* S_out,
                        const float* mu_other, const float* S_other, float* mu_in, float* S_in,
                        unsigned flags);
/* BayesBase.prod(::MvNormal, ::MvNormal) in (xi, W): (xi1 + xi2, W1 + W2)
 * [ref: fold at src/model/plugins/reactivemp_inference.jl:365-374]                              */
int rxg_prod_gaussian_f32(rxg_ctx*, int64_t n, int d, const float* xi1, const float* W1,
                          const float* xi2, const float* W2, float* xi, float* W, unsigned flags);
/* weightedmean_precision(::MvNormalMeanCovariance) / mean_cov(::MvNormalWeightedMeanPrecision):
 * one Cholesky SPD inverse each (FastCholesky.cholinv) [ref: re-export src/RxInfer.jl:6]        */
int rxg_meancov_to_wmp_f32(rxg_ctx*, int64_t n, int d, const float* mu, const float* S, float* xi,
                           float* W, int32_t* status, unsigned flags);
int rxg_wmp_to_meancov_f32(rxg_ctx*, int64_t n, int d, const float* xi, const float* W, float* mu,
                           float* S, int32_t* status, unsigned flags);
/* Marginal at a random variable: product of k inbound (xi, W) messages then mean_cov
 * [ref: src/model/plugins/reactivemp_inference.jl:370-455]; xi_list/W_list are arrays of k
 * HOST-resident pointers to the message buffers.                                                */
int rxg_marginal_gaussian_f32(rxg_ctx*, int64_t n, int d, int k, const float* const* xi_list,
                              const float* const* W_list, float* mu, float* S, int32_t* status,
                              unsigned flags);

/* Univariate / Gamma-precision VMP rules (SURVEY.md 8a rows 8-9)
 * @rule NormalMeanPrecision(:tau)(q_out, q_mu) -> GammaShapeRate(3/2, ((m_o-m_m)^2+v_o+v_m)/2)
 * [ref: test/models/aliases/aliases_gamma_tests.jl:13-18]                                        */
int rxg_rule_normal_precision_tau_f32(rxg_ctx*, int64_t n, const float* m_out, const float* v_out,
                                      const float* m_mu, const float* v_mu, float* shape,
                                      float* rate, unsigned flags);
/* @rule NormalMeanPrecision(:out)(m_mu, q_tau) -> N(m_mu, v_mu + rate/shape)                    */
int rxg_rule_normal_precision_out_f32(rxg_ctx*, int64_t n, const float* m_mu, const float* v_mu,
                                      const float* shape, const float* rate, float* m_out,
                                      float* v_out, unsigned flags);
/* structured variant (q_out_mu jointly Gaussian, m_joint[2][n], V_joint[2][2][n]): GammaShapeRate(3/2,
 * 1/2 [V11 + V22 - V12 - V21 + (m1 - m2)^2])  (upstream rules/normal_mean_precision/precision.jl)              */
int rxg_rule_normal_precision_tau_joint_f32(rxg_ctx*, int64_t n, const float* m_joint, const float* V_joint,
                                            float* shape, float* rate, unsigned flags);
/* Wishart precision -- the multivariate twin of the Gamma rules, in the WishartFast parametrisation (df, INVERSE
 * scale) so that products are additions [ref: test/models/iid/mv_iid_precision_tests.jl:10-41]:
 * @rule MvNormalMeanPrecision(:Lambda)(q_out, q_mu) -> Wishart(d + 2, inv(V_out + V_mu + (m_out - m_mu)(m_out - m_mu)'))  */
int rxg_rule_mvnormal_precision_lambda_f32(rxg_ctx*, int64_t n, int d, const float* m_out, const float* V_out,
                                           const float* m_mu, const float* V_mu, float* df, float* inv_scale,
                                           unsigned flags);
/* prod(Wishart, Wishart) = Wishart(df1 + df2 - d - 1, inv(inv(S1) + inv(S2)))                                   */
int rxg_prod_wishart_f32(rxg_ctx*, int64_t n, int d, const float* df1, const float* inv_scale1, const float* df2,
                         const float* inv_scale2, float* df, float* inv_scale, unsigned flags);
/* mean(Wishart(df, S)) = df * S = df * inv(inv_scale); status[n] optional                                      */
int rxg_wishart_mean_f32(rxg_ctx*, int64_t n, int d, const float* df, const float* inv_scale, float* mean,
                         int32_t* status, unsigned flags);
/* Fused mean-field VMP of the multivariate IID model with unknown mean and precision, `batch` independent data sets:
 *   m ~ MvNormal(mu0, inv(Lambda0)),  P ~ Wishart(nu0, inv(inv_scale0)),  y[i] ~ MvNormal(m, inv(P)),  q(m) q(P)
 * [ref: model, constraints and initialisation test/models/iid/mv_iid_precision_tests.jl:10-41].  y[N][d][batch];
 * init_E_P[d][d] = mean of the initial q(P) (host); outputs q(m) = (m_mean[d][batch], m_cov[d][d][batch]),
 * q(P) = Wishart(df[batch], inv(inv_scale[d][d][batch])).  d <= 6 (d = 7.. -> RXG_ERR_UNSUPPORTED); d, N, iterations
 * >= 1 and nu0 > d - 1, else RXG_ERR_BAD_ARG.  Device pointers (RXG_ERR_UNSUPPORTED otherwise).                  */
int rxg_mv_iid_wishart_vmp_f32(rxg_ctx*, int d, int N, int64_t batch, int iterations, const float* mu0,
                               const float* Lambda0, float nu0, const float* inv_scale0, const float* init_E_P,
                               const float* y, float* m_mean, float* m_cov, float* df, float* inv_scale,
                               int32_t* status, unsigned flags);
/* Fused mean-field VMP of the reference's autoregressive regression model, `batch` independent series:
 *   gamma ~ Gamma(a0, b0), theta ~ MvNormal(0, I / theta_prior_precision), y[i] ~ Normal(dot(x[i], theta), 1 / gamma),
 *   x[i] = (s[i-1], ..., s[i-order]) lags of the series itself, q(gamma) q(theta), q(gamma) initialised to
 *   Gamma(init_shape, init_rate) [ref: test/models/autoregressive/ar_tests.jl:7-36].  series[N][batch]; outputs
 *   theta_mean[order][batch], theta_cov[order][order][batch], gamma_shape / gamma_rate[batch], free_energy[iterations][batch]
 *   or NULL (Bethe free energy after every iteration, in fp64: the reference asserts it to decrease, :69-70, and the
 *   decreases are ~1e-5 on values of ~1.4e3).  order <= 8.                                                         */
int rxg_ar_vmp_f32(rxg_ctx*, int order, int N, int64_t batch, int iterations, float a0, float b0,
                   float theta_prior_precision, float init_shape, float init_rate, const float* series,
                   float* theta_mean, float* theta_cov, float* gamma_shape, float* gamma_rate,
                   double* free_energy, unsigned flags);
/* Fused structured VMP of the reference's LATENT autoregressive model, `batch` independent series, one launch:
 *   gamma ~ Gamma(a0, b0); theta ~ N(0, I / w0); x0 ~ N(0, I / p0); x[t] ~ AR(x[t-1], theta, gamma) with
 *   ARMeta(Multivariate | Univariate, order, ARsafe()); y[t] ~ Normal(dot(c, x[t]), 1 / tau), c = e1 (ReactiveMP.ar_unit);
 *   q(x, x0) q(gamma) q(theta); q(gamma), q(theta) initialised to Gamma(init_shape, init_rate), N(0, I / init_theta_precision)
 *   [ref: test/models/autoregressive/lar_tests.jl:52-122; free-energy pins :170 (AR(1): 518.9182342) and :201 (AR(5): 514.66086)].
 *   The Univariate AR(1) node is the order = 1 case.  params (HOST, 8 floats, all > 0) = {tau, a0, b0, w0, p0, init_shape,
 *   init_rate, init_theta_precision}.  y[T][batch]; outputs: x_mean[T][order][batch], x_cov[T][order][order][batch] of the
 *   LAST iteration (KeepLast; either may be NULL), theta_mean[iterations][order][batch],
 *   theta_cov[iterations][order][order][batch], gamma_shape / gamma_rate[iterations][batch] (KeepEach),
 *   free_energy[iterations][batch] in fp64 or NULL, status[batch] or NULL.  Every iteration is a covariance-form filter + RTS
 *   smoother over the companion-matrix state space in the exact limit of the AR node's deterministic coordinates (the
 *   reference regularises them with a precision of 1e12), fp32 recursions, fp64 statistics / parameter updates / free energy.
 *   order <= 6.  Device pointers.                                                                                   */
int rxg_lar_vmp_f32(rxg_ctx*, int order, int T, int64_t batch, int iterations, const float* params, const float* y,
                    float* x_mean, float* x_cov, float* theta_mean, float* theta_cov, float* gamma_shape,
                    float* gamma_rate, double* free_energy, int32_t* status, unsigned flags);
/* Fused mean-field VMP of the Gaussian mixture model, `batch` independent data sets, all iterations in one launch:
 *   s ~ Dirichlet(alpha0), m[k] ~ MvNormal(mu0[k], V0[k]), W[k] ~ Wishart(nu0[k], S0[k]) (precision; S0 the scale),
 *   z[i] ~ Categorical(s), y[i] ~ NormalMixture(z[i], m, W), q(s) prod q(m[k]) prod q(W[k]) prod q(z[i]), initialised to
 *   Dirichlet(alpha_init), MvNormal(m_init[k], Vm_init[k]), Wishart(nu_init[k], S_init[k])
 *   [ref: test/models/mixtures/gmm_multivariate_tests.jl:4-24, :37-64; gmm_univariate_tests.jl:6-26 is the d = 1, K = 2
 *   case with Beta(a, b) = Dirichlet([a, b]) and Gamma(shape, rate) = Wishart(2 shape, 1 / (2 rate))].  Priors and initial
 *   marginals are HOST arrays shared by every chain: alpha0[K], mu0[K][d], V0[K][d][d], nu0[K], S0[K][d][d], likewise the
 *   *_init.  y[N][d][batch].  Outputs of the last iteration: alpha[K][batch], m_mean[K][d][batch], m_cov[K][d][d][batch],
 *   w_df[K][batch], w_inv_scale[K][d][d][batch] (q(W[k]) = Wishart(w_df, inv(w_inv_scale))).  Optional (NULL = not
 *   wanted): free_energy[iterations][batch] (fp64, Bethe free energy after every iteration), z_prob[N][K][batch] (q(z) of
 *   the last iteration), the KeepEach histories hist_alpha[iterations][K][batch], hist_m_mean[iterations][K][d][batch],
 *   hist_m_cov[iterations][K][d][d][batch], hist_w_df[iterations][K][batch], hist_w_inv_scale[iterations][K][d][d][batch],
 *   status[batch] (RXG_ERR_NOT_SPD for a chain whose update met a non-SPD matrix).  Per iteration: q(z), then q(m[k]) with
 *   the previous E[W[k]], q(W[k]) with the new q(m[k]), q(s).  1 <= d <= 4 and 2 <= K <= 8, else RXG_ERR_UNSUPPORTED;
 *   N, batch, iterations >= 1, alpha0 and alpha_init > 0, nu0 and nu_init > d - 1, V0, S0, Vm_init, S_init symmetric
 *   positive definite, else RXG_ERR_BAD_ARG.  Device pointers (RXG_ERR_UNSUPPORTED otherwise).                        */
int rxg_gmm_vmp_f32(rxg_ctx*, int d, int K, int N, int64_t batch, int iterations, const float* alpha0, const float* mu0,
                    const float* V0, const float* nu0, const float* S0, const float* alpha_init, const float* m_init,
                    const float* Vm_init, const float* nu_init, const float* S_init, const float* y, float* alpha,
                    float* m_mean, float* m_cov, float* w_df, float* w_inv_scale, double* free_energy, float* z_prob,
                    float* hist_alpha, float* hist_m_mean, float* hist_m_cov, float* hist_w_df, float* hist_w_inv_scale,
                    int32_t* status, unsigned flags);
/* Fused structured VMP of the hidden Markov model, `batch` independent chains, all iterations in one launch:
 *   A ~ DirichletCollection(A_prior) (K x K, column j = p(s_t | s_{t-1} = j)), B ~ DirichletCollection(B_prior) (M x K,
 *   column j = p(x_t | s_t = j)), s_0 ~ Categorical(p0), s[t] ~ DiscreteTransition(s[t-1], A), x[t] ~
 *   DiscreteTransition(s[t], B), q(s, s_0) q(A) q(B), initialised to DirichletCollection(A_init), (B_init)
 *   [ref: test/models/statespace/hmm_tests.jl:8-45; a known A as in test/inference/inference_tests.jl:2062-2088].  Either
 *   matrix is learned (prior and init non-NULL, its *_known NULL) or known (*_known, a probability matrix, the other two
 *   NULL).  Host arrays shared by every chain, row-major [row][column] (row = next state or symbol, column = conditioning
 *   state): p0[K], A_*[K][K], B_*[M][K].  x[T][batch] uint8 symbols 0..M-1, 255 = missing (a pure transition step).
 *   Outputs: s_prob[T][K][batch] (q(s_t) of the last iteration; also the forward stash), and optional (NULL = not wanted):
 *   s0_prob[K][batch], A_alpha[K][K][batch] / B_alpha[M][K][batch] (of a learned matrix), free_energy[iterations][batch]
 *   (fp64, Bethe free energy after every iteration; -log p(x) with both matrices known), the KeepEach histories
 *   hist_s[iterations][T][K][batch], hist_A[iterations][K][K][batch], hist_B[iterations][M][K][batch], status[batch]
 *   (RXG_ERR_BAD_ARG for a chain with a symbol >= M other than 255, read as missing; RXG_ERR_NAN for a chain whose data are
 *   impossible under its model).  Per iteration: forward-backward with the previous q(A), q(B), then both updated.
 *   2 <= K <= 8 and 2 <= M <= 16, else RXG_ERR_UNSUPPORTED; T, batch, iterations >= 1, Dirichlet parameters > 0, p0 and
 *   the columns of a known matrix non-negative with sum 1 (within 1e-5), else RXG_ERR_BAD_ARG.  Device pointers
 *   (RXG_ERR_UNSUPPORTED otherwise).                                                                                  */
int rxg_hmm_vmp_f32(rxg_ctx*, int K, int M, int T, int64_t batch, int iterations, const float* p0, const float* A_prior,
                    const float* A_init, const float* A_known, const float* B_prior, const float* B_init,
                    const float* B_known, const uint8_t* x, float* s_prob, float* s0_prob, float* A_alpha, float* B_alpha,
                    double* free_energy, float* hist_s, float* hist_A, float* hist_B, int32_t* status, unsigned flags);
/* Fused structured VMP of the hidden Markov model with Gaussian emissions, `batch` independent chains, all iterations in one
 *   launch: A ~ DirichletCollection(A_prior) (K x K, column j = p(s_t | s_{t-1} = j)) or a known probability matrix,
 *   m[k] ~ MvNormal(mu0[k], V0[k]), W[k] ~ Wishart(nu0[k], S0[k]) (precision; S0 the scale), s_0 ~ Categorical(p0),
 *   s[t] ~ DiscreteTransition(s[t-1], A), y[t] ~ NormalMixture(switch = s[t], m, W), q(s_0, s) q(A) prod q(m[k]) q(W[k]),
 *   initialised to DirichletCollection(A_init), MvNormal(m_init[k], Vm_init[k]), Wishart(nu_init[k], S_init[k])
 *   [ref: test/models/statespace/hmm_tests.jl:8-45 (the chain, DiscreteTransition and its structured factorisation) with
 *   the NormalMixture emission of test/models/mixtures/gmm_multivariate_tests.jl:4-24; no reference test runs this model,
 *   so nothing pins it (DESIGN 3.20)].  A is learned (A_prior and A_init non-NULL, A_known NULL) or known (A_known, the
 *   other two NULL).  Host arrays shared by every chain, row-major: p0[K], A_*[K][K] (row = next state), mu0[K][d],
 *   V0[K][d][d] (covariance), nu0[K], S0[K][d][d], likewise m_init, Vm_init, nu_init, S_init.  y[T][d][batch]; a step whose
 *   d components are all NaN is missing (a pure transition).  Outputs: s_prob[T][K][batch] (q(s_t) of the last iteration;
 *   also the forward stash), and optional (NULL = not wanted): s0_prob[K][batch], A_alpha[K][K][batch] (A learned),
 *   m_mean[K][d][batch], m_cov[K][d][d][batch], w_df[K][batch], w_inv_scale[K][d][d][batch] (q(W[k]) = Wishart(w_df,
 *   inv(w_inv_scale))), free_energy[iterations][batch] (fp64, Bethe free energy after every iteration), the KeepEach
 *   histories hist_s[iterations][T][K][batch], hist_A[iterations][K][K][batch], hist_m_mean[iterations][K][d][batch],
 *   hist_m_cov[iterations][K][d][d][batch], hist_w_df[iterations][K][batch], hist_w_inv_scale[iterations][K][d][d][batch],
 *   status[batch] (RXG_ERR_BAD_ARG for a chain with a non-finite datum other than an all-NaN step, read as missing;
 *   RXG_ERR_NAN for a chain whose normaliser vanished; RXG_ERR_NOT_SPD for a chain whose update met a non-SPD matrix).
 *   Per iteration: forward-backward with the previous q(A), q(m), q(W), then q(A), q(m[k]) with the previous E[W[k]],
 *   q(W[k]) with the new q(m[k]).  1 <= d <= 4 and 2 <= K <= 8, else RXG_ERR_UNSUPPORTED; T, batch, iterations >= 1,
 *   Dirichlet parameters > 0, p0 and the columns of A_known probability vectors (within 1e-5), nu0 and nu_init > d - 1,
 *   V0, S0, Vm_init, S_init symmetric positive definite, else RXG_ERR_BAD_ARG.  Device pointers (RXG_ERR_UNSUPPORTED
 *   otherwise).                                                                                                        */
int rxg_hmm_gauss_vmp_f32(rxg_ctx*, int d, int K, int T, int64_t batch, int iterations, const float* p0,
                          const float* A_prior, const float* A_init, const float* A_known, const float* mu0, const float* V0,
                          const float* nu0, const float* S0, const float* m_init, const float* Vm_init, const float* nu_init,
                          const float* S_init, const float* y, float* s_prob, float* s0_prob, float* A_alpha, float* m_mean,
                          float* m_cov, float* w_df, float* w_inv_scale, double* free_energy, float* hist_s, float* hist_A,
                          float* hist_m_mean, float* hist_m_cov, float* hist_w_df, float* hist_w_inv_scale,
                          int32_t* status, unsigned flags);
/* Bayesian binomial / logistic regression, mean-field Polya-Gamma VMP, `batch` independent chains, all iterations in one
 *   launch: beta ~ MvNormalWeightedMeanPrecision(xi0, W0), y[i] ~ BinomialPolya(x[i], n[i], beta) (y[i] ~ Binomial(n[i],
 *   sigmoid(x[i]' beta))), i = 1..N, q(beta) Gaussian [ref: test/models/regression/binomialreg_tests.jl:32-43; the rule
 *   reads q(beta) where the reference may read the cavity, and the reference pins no free energy (DESIGN 3.21)].  Host
 *   arrays shared by every chain: xi0[p], W0[p][p] (symmetric positive definite).  X[N][p][batch] fp32, y[N][batch] int32,
 *   ntrials[N][batch] int32 or NULL (every n = 1: logistic regression); a sample with n = 0 contributes nothing (padding
 *   of ragged batches).  Outputs: beta_mean[p][batch], and optional (NULL = not wanted): beta_cov[p][p][batch],
 *   free_energy[iterations][batch] (fp64, the collapsed Polya-Gamma bound of the posterior each iteration returns), the
 *   KeepEach histories hist_mean[iterations][p][batch], hist_cov[iterations][p][p][batch], status[batch] (RXG_ERR_BAD_ARG
 *   for a chain with a sample with a non-finite x, y < 0, n < 0 or y > n, read as n = 0; RXG_ERR_NOT_SPD for a
 *   non-positive pivot; RXG_ERR_NAN for a non-finite result; the last two take precedence).  1 <= p <= 8, else
 *   RXG_ERR_UNSUPPORTED; N, batch, iterations >= 1, finite xi0 and W0 symmetric positive definite, else RXG_ERR_BAD_ARG.
 *   Device pointers (RXG_ERR_UNSUPPORTED otherwise).  RXG_OPT_POLYA_PATH selects the kernel.                           */
int rxg_binomial_polya_vmp_f32(rxg_ctx*, int p, int N, int64_t batch, int iterations, const float* xi0, const float* W0,
                               const float* X, const int32_t* y, const int32_t* ntrials, float* beta_mean, float* beta_cov,
                               double* free_energy, float* hist_mean, float* hist_cov, int32_t* status, unsigned flags);
/* Bayesian multinomial regression, mean-field Polya-Gamma VMP, `batch` independent chains, all iterations in one call:
 *   psi ~ MvNormalWeightedMeanPrecision(xi0, W0), y[i] ~ MultinomialPolya(N_i, psi), i = 1..n, N_i = sum_k y[i][k], read
 *   through stick-breaking (y_ik ~ Binomial(N_ik, sigmoid(psi_k)), N_ik = sum_{j >= k} y_ij), D = K - 1, q(psi) Gaussian
 *   [ref: test/models/regression/multinomialreg_tests.jl; the rule reads q(psi) where the reference may read the cavity
 *   (DESIGN 3.22)].  Host arrays shared by every chain: xi0[D], W0[D][D] (symmetric positive definite).  y[n][K][batch]
 *   int32 counts; an all-zero sample contributes nothing (padding of ragged batches).  Outputs: psi_mean[D][batch], and
 *   optional (NULL = not wanted): psi_cov[D][D][batch], free_energy[iterations][batch] (fp64, the collapsed Polya-Gamma
 *   bound of the posterior each iteration returns), the KeepEach histories hist_mean[iterations][D][batch],
 *   hist_cov[iterations][D][D][batch], status[batch] (RXG_ERR_BAD_ARG for a chain with a negative count, that sample read
 *   as all-zero; RXG_ERR_NOT_SPD for a non-positive pivot; RXG_ERR_NAN for a non-finite result; the last two take
 *   precedence).  2 <= K <= 64, else RXG_ERR_UNSUPPORTED; n, batch, iterations >= 1, finite xi0 and W0 symmetric
 *   positive definite, else RXG_ERR_BAD_ARG.  Device pointers (RXG_ERR_UNSUPPORTED otherwise).  Two kernel launches.   */
int rxg_multinomial_polya_vmp_f32(rxg_ctx*, int K, int n, int64_t batch, int iterations, const float* xi0, const float* W0,
                                  const int32_t* y, float* psi_mean, float* psi_cov, double* free_energy, float* hist_mean,
                                  float* hist_cov, int32_t* status, unsigned flags);
/* The same model online (@autoupdates of q(psi), one datum at a time): datum t of y[T][K][batch] runs `iterations` steps
 *   from the base q_{t-1}, then q_t is the next base.  The carry is fp64: m_in[D][batch], S_in[D][D][batch] (both NULL:
 *   every chain starts at N(W0^-1 xi0, W0^-1)), m_out, S_out the same shapes (may be m_in, S_in: updated in place), so a
 *   stream split into chunks gives the bits of one call.  Optional per datum: hist_mean[T][D][batch],
 *   hist_cov[T][D][D][batch], free_energy[T][batch] (fp64, KL(q_t || q_{t-1}) minus the bound of datum t's evidence:
 *   free_energy_final_only_history), status[batch] as above.  Limits and errors as rxg_multinomial_polya_vmp_f32.     */
int rxg_multinomial_polya_online_f32(rxg_ctx*, int K, int T, int64_t batch, int iterations, const float* xi0, const float* W0,
                                     const double* m_in, const double* S_in, const int32_t* y, double* m_out, double* S_out,
                                     float* hist_mean, float* hist_cov, double* free_energy, int32_t* status,
                                     unsigned flags);
/* prod(GammaShapeRate, GammaShapeRate) = (a1 + a2 - 1, b1 + b2)                                 */
int rxg_prod_gamma_f32(rxg_ctx*, int64_t n, const float* a1, const float* b1, const float* a2,
                       const float* b2, float* a, float* b, unsigned flags);
/* prod of two univariate Normals in (mean, variance) I/O                                        */
int rxg_prod_normal_f32(rxg_ctx*, int64_t n, const float* m1, const float* v1, const float* m2,
                        const float* v2, float* m, float* v, unsigned flags);

/* GCV node rules (SURVEY.md 8a row 10) [ref: test/models/statespace/hgf_tests.jl:10-40;
 * formulas restated at test/inference/inference_tests.jl:587-607]; kappa, omega PointMass.
 * @rule GCV(:y)(m_x, q_z, ...) -> N(m_x, v_x + 1/(A B))  (and symmetric :x)                     */
int rxg_rule_gcv_out_f32(rxg_ctx*, int64_t n, const float* m_x, const float* v_x,
                         const float* m_z, const float* v_z, float kappa, float omega,
                         float* m_out, float* v_out, unsigned flags);
/* @marginalrule GCV(:y_x) -> joint (m[2][n], V[2][2][n])                                        */
int rxg_marginalrule_gcv_yx_f32(rxg_ctx*, int64_t n, const float* m_y, const float* v_y,
                                const float* m_x, const float* v_x, const float* m_z,
                                const float* v_z, float kappa, float omega, float* m, float* V,
                                unsigned flags);
/* @rule GCV(:z)(q_y_x, ...) -> ExponentialLinearQuadratic(a,b,c,d), then prod(Normal prior, ELQ)
 * by GaussHermiteCubature(31) moment matching -> q(z) = N(m_z, v_z)                             */
int rxg_rule_gcv_z_prod_f32(rxg_ctx*, int64_t n, const float* m_yx, const float* V_yx,
                            const float* m_zprior, const float* v_zprior, float kappa, float omega,
                            float* m_z, float* v_z, unsigned flags);

/* ------------------------------------------------------------------ fused whole-chain sweeps --
 * Replace, for the batched case, the Rocket-driven schedule + per-message dispatch that one
 * infer(model = linear_gaussian_ssm_smoothing(...), data = (y = ...,)) executes
 * [ref: iteration loop src/inference/batch.jl:391-430; model benchmarks/...ipynb:95-105;
 *  test/models/statespace/mlgssm_test.jl:8-17].  One launch runs the forward sweep t = 1..T and
 * the backward sweep t = T..1 for `batch` independent chains: 6 rule messages + 2 products +
 * 1 marginal per (chain, step).
 *
 *   x[1] ~ N(m0, S0);  x[t] ~ N(A x[t-1] + u, P);  y[t] ~ N(B x[t], Q)     (A d x d, B m x d)
 *
 * `u` (d floats, or NULL for none) is a constant transition offset: the `+` rule with a PointMass
 * operand fused into the sweep [ref: `x[i] ~ x_prev + c`, test/models/statespace/
 * ulgssm_tests.jl:12].  With RXG_TRANSITION_FIRST the prior sits on the state BEFORE x[1]
 * (x_prior ~ N(m0, S0); x[1] ~ N(A x_prior + u, P)), as in test/models/statespace/
 * mlgssm_test.jl:8-17 and the notebook's one-step filtering model (ipynb:110-113).
 *
 * Inputs : y[T][m][batch]; ymask[T][batch] (uint8, 1 = observed) or NULL
 *          [ref: missing data semantics docs/src/manuals/inference/static.md:98-125];
 *          A,B,P,Q,m0,S0,u row-major, shared HOST arrays (or device [..][batch] arrays with
 *          RXG_MODEL_PER_CHAIN).
 *          With RXG_U_SEQ_SHARED / RXG_U_SEQ_CHAIN, u is a per-step input sequence of T rows instead
 *          (u[T][d] host, or u[T][d][batch] device; see the flags): x[t] ~ N(A x[t-1] + u[t], P).
 * Outputs: post_mean[T][d][batch], post_cov[T][d][d][batch]  (== posteriors[:x], as
 *          MvNormalMeanCovariance) [ref: src/inference/batch.jl:475-481];
 *          neg_log_evidence[batch] or NULL (== Bethe free energy on this tree
 *          [ref: src/model/plugins/reactivemp_free_energy.jl:84-126]);
 *          status[batch] or NULL (per-chain RXG_OK / RXG_ERR_NOT_SPD / RXG_ERR_NAN).
 * post_mean / post_cov double as the forward->backward stash (no extra workspace).             */
int rxg_lgssm_smooth_f32(rxg_ctx*, int d, int m, int T, int64_t batch, const float* A,
                         const float* B, const float* P, const float* Q, const float* m0,
                         const float* S0, const float* u, const float* y, const uint8_t* ymask,
                         float* post_mean, float* post_cov, float* neg_log_evidence,
                         int32_t* status, unsigned flags);
/* Smoothing sweep + predictive distributions of the observations (result.predictions)
 * [ref: predictvars and the automatic predictions for data containing `missing`, src/inference/batch.jl:203-246;
 *  tested in test/inference/prediction_tests.jl:193-420].  The prediction for y[t] is the reference's message
 * toward y[t]: the cavity fwd_t x bwd_t passed through *(:out) with B and MvNormalMeanCovariance(:out) with Q.
 * With the smoothed posterior (mu_s, S_s) and D_t = Q - B S_s[t] B' (formed and factorised in fp64):
 *     missing y[t]:   N(B mu_s[t], B S_s[t] B' + Q)
 *     observed y[t]:  N(y_t - Q D_t^-1 (y_t - B mu_s[t]), Q D_t^-1 Q)
 *     forecast k = 1..H from (x_0, S_0) = (mu_s[T-1], S_s[T-1]):  x_k = A x_{k-1} + u, S_k = A S_{k-1} A' + P,
 *                     prediction N(B x_k, B S_k B' + Q)  (== the smoother on y padded with H missing steps)
 * Arguments shared with rxg_lgssm_smooth_f32 mean the same, and post_mean / post_cov / neg_log_evidence are
 * bit-identical to its outputs.  Outputs: pred_mean[T+H][m][batch] (rows T.. are the forecasts), pred_cov
 * [T+H][m][m][batch] ([T+H][m][m] with RXG_COV_SHARED_OUT) or NULL, fc_mean[H][d][batch] (state forecasts) or
 * NULL, fc_cov[H][d][d][batch] ([H][d][d] with RXG_COV_SHARED_OUT) or NULL.  post_cov may be NULL (shared model,
 * no per-chain mask) only at the register-resident shapes, whose own covariance table then feeds the post-pass; other
 * shapes return RXG_ERR_UNSUPPORTED before anything runs.  Device pointers only
 * (RXG_ERR_UNSUPPORTED otherwise); H < 0 or pred_mean NULL -> RXG_ERR_BAD_ARG; a chain whose D_t is not SPD gets
 * RXG_ERR_NOT_SPD in status[b] (shared model: every chain, and the call returns RXG_ERR_NOT_SPD).  As for the
 * smoother, y at masked steps is ignored but must be finite.
 * With RXG_U_SEQ_SHARED / RXG_U_SEQ_CHAIN the input sequence has T + H rows: forecast k = 1..H steps
 * x_k = A x_{k-1} + u[T + k - 1].  The predictions at steps t < T depend only on (y, mu_s, S_s).  */
int rxg_lgssm_smooth_predict_f32(rxg_ctx*, int d, int m, int T, int H, int64_t batch, const float* A,
                                 const float* B, const float* P, const float* Q, const float* m0,
                                 const float* S0, const float* u, const float* y, const uint8_t* ymask,
                                 float* post_mean, float* post_cov, float* neg_log_evidence,
                                 float* pred_mean, float* pred_cov, float* fc_mean, float* fc_cov,
                                 int32_t* status, unsigned flags);
/* Forward half only (filtering) -- what the streaming engine computes per datum with
 * @autoupdates x_min_t_mean, x_min_t_cov = mean_cov(q(x_t))
 * [ref: src/inference/streaming.jl:344-388; src/inference/autoupdates.jl:614-659; ipynb:199-216].
 * RXG_U_SEQ_SHARED / RXG_U_SEQ_CHAIN as for rxg_lgssm_smooth_f32 (T rows).                        */
int rxg_lgssm_filter_f32(rxg_ctx*, int d, int m, int T, int64_t batch, const float* A,
                         const float* B, const float* P, const float* Q, const float* m0,
                         const float* S0, const float* u, const float* y, const uint8_t* ymask,
                         float* filt_mean, float* filt_cov, float* neg_log_evidence,
                         int32_t* status, unsigned flags);
/* VMP around the smoother with an unknown observation precision shared over time, one per chain
 * (d = m = 1): y[t] ~ N(x[t], 1/tau), tau ~ Gamma(a0, b0), q(x) q(tau)
 * [ref: rules of test/models/aliases/aliases_gamma_tests.jl; use case
 *  test/callbacks/benchmark_tests.jl:8-37].  y[T][batch]; outputs post_mean/var[T][batch],
 * shape/rate[batch].  T, iterations >= 1 and v_proc, v0, a0, b0, init_E_tau > 0, else
 * RXG_ERR_BAD_ARG.  Device pointers (RXG_ERR_UNSUPPORTED otherwise).                            */
int rxg_lgssm_vmp_gamma_f32(rxg_ctx*, int T, int64_t batch, int iterations, float a, float v_proc,
                            float m0, float v0, float a0, float b0, float init_E_tau,
                            const float* y, float* post_mean, float* post_var, float* shape,
                            float* rate, unsigned flags);
/* Same with the Bethe free energy after every iteration, free_energy[iterations][batch] (or NULL)
 * [ref: free_energy = true, src/inference/batch.jl:184-189; definition src/model/plugins/reactivemp_free_energy.jl:84-126]. */
int rxg_lgssm_vmp_gamma_fe_f32(rxg_ctx*, int T, int64_t batch, int iterations, float a, float v_proc,
                               float m0, float v0, float a0, float b0, float init_E_tau, const float* y,
                               float* post_mean, float* post_var, float* shape, float* rate,
                               float* free_energy, unsigned flags);
/* VMP around the multivariate smoother with an unknown observation precision MATRIX w, one per chain
 * [ref: docs/src/manuals/model-specification.md:265-271, run with constraints = q(x, w) = q(x)q(w) and `iterations`]:
 *   w ~ Wishart(nu0, inv(inv_scale0)); x[1] ~ N(m0, S0) (RXG_TRANSITION_FIRST: one transition earlier);
 *   x[t] ~ N(A x[t-1] + u, P); y[t] ~ N(B x[t], inv(w)); q(x) q(w), q(x) structured over the chain.
 * A, B, P, m0, S0, u (constant, [d] or NULL), inv_scale0 and init_E_W (= E[w] of the initial q(w)) are HOST arrays shared
 * by all chains; the data and outputs are device arrays (RXG_PTR_DEVICE is required).  y[T][m][batch]; ymask NULL,
 * [T][batch] (device) or, with RXG_MASK_SHARED, one host pattern [T].  Outputs: q(x) of the LAST iteration (KeepLast)
 * in post_mean[T][d][batch] / post_cov[T][d][d][batch]; q(w) = Wishart(df, inv(inv_scale)) after EVERY iteration
 * (KeepEach) in df[iterations][batch] / inv_scale[iterations][m][m][batch]; the Bethe free energy after every iteration
 * in fp64, free_energy[iterations][batch] or NULL; status[batch] or NULL (RXG_ERR_NOT_SPD when a pivot of the chain's
 * recursion or Wishart update was not positive).  Each iteration runs the Kalman filter + RTS smoother with
 * Q = inv(E[w]), then q(w) = (nu0 + N_b, inv_scale0 + sum_observed (y - B mu)(y - B mu)' + B Sigma B').
 * d, m in 1..6.  Flags: RXG_PTR_DEVICE, RXG_TRANSITION_FIRST, RXG_MASK_SHARED, RXG_ASYNC; others are refused with
 * RXG_ERR_UNSUPPORTED (the covariances depend on the chain through w).  iterations >= 1, nu0 > m - 1, and SPD
 * inv_scale0 / init_E_W, else RXG_ERR_BAD_ARG.                                                                  */
int rxg_lgssm_vmp_wishart_f32(rxg_ctx*, int d, int m, int T, int64_t batch, int iterations, const float* A,
                              const float* B, const float* P, const float* m0, const float* S0, const float* u,
                              float nu0, const float* inv_scale0, const float* init_E_W, const float* y,
                              const uint8_t* ymask, float* post_mean, float* post_cov, float* df, float* inv_scale,
                              double* free_energy, int32_t* status, unsigned flags);
/* The same VMP with an unknown PROCESS precision matrix w_p, alone or together with the observation precision w_q:
 *   w_p ~ Wishart(nu_p0, inv(inv_scale_p0)) (else P known); w_q ~ Wishart(nu_q0, inv(inv_scale_q0)) (else Q known);
 *   x[1] ~ N(m0, S0) (RXG_TRANSITION_FIRST: one transition earlier); x[t] ~ N(A x[t-1] + u, inv(w_p));
 *   y[t] ~ N(B x[t], inv(w_q)); q(x) q(w_p) q(w_q), q(x) structured over the chain.
 * For each noise pass exactly one of the known matrix (P / Q) and the pair (inv_scale_0, init_E_W = E[w] of the initial
 * q(w)); at least one noise is learned (both known is the plain smoother: RXG_ERR_BAD_ARG).  A learned noise needs its
 * outputs df_*[iterations][batch] / inv_scale_*[iterations][k][k][batch] (k = d for p, m for q, after EVERY iteration);
 * a known noise's outputs must be NULL.  Each iteration runs the Kalman filter + RTS smoother with P = inv(E[w_p]) and
 * Q = inv(E[w_q]), then q(w_p) = (nu_p0 + T - 1 + tf, inv_scale_p0 + R_p) with R_p the sum over the transitions of
 * E[(x[t+1] - A x[t] - u)(x[t+1] - A x[t] - u)'] under the pairwise smoothed marginal (masks do not change the count),
 * and q(w_q) as rxg_lgssm_vmp_wishart_f32 updates it.  free_energy[iterations][batch] (fp64) or NULL: the Bethe free
 * energy with one Wishart block per learned noise.  Host model arrays, device data, masks, status, flags, d, m in 1..6
 * and the refusals as rxg_lgssm_vmp_wishart_f32; nu_p0 > d - 1, nu_q0 > m - 1 and SPD inverse scales / initial E[w]
 * of the learned noises, else RXG_ERR_BAD_ARG.  Called with Q learned and P known it computes exactly what
 * rxg_lgssm_vmp_wishart_f32 computes.                                                                          */
int rxg_lgssm_vmp_noise_f32(rxg_ctx*, int d, int m, int T, int64_t batch, int iterations, const float* A, const float* B,
                            const float* m0, const float* S0, const float* u, const float* P, float nu_p0,
                            const float* inv_scale_p0, const float* init_E_Wp, const float* Q, float nu_q0,
                            const float* inv_scale_q0, const float* init_E_Wq, const float* y, const uint8_t* ymask,
                            float* post_mean, float* post_cov, float* df_p, float* inv_scale_p, float* df_q,
                            float* inv_scale_q, double* free_energy, int32_t* status, unsigned flags);
/* The same VMP that also learns the TRANSITION MATRIX per chain (RxInfer's ContinuousTransition node with a Gaussian
 * prior on a = vec(A), reshaped linearly to A):
 *   a ~ N(a_mean0, a_cov0); w_p ~ Wishart(nu_p0, inv(inv_scale_p0)) (else P known); w_q likewise (else Q known);
 *   x[1] ~ N(m0, S0) (RXG_TRANSITION_FIRST: one transition earlier); x[t] ~ N(A x[t-1] + u, inv(w_p));
 *   y[t] ~ N(B x[t], inv(w_q)); q(x) q(a) q(w_p) q(w_q), q(x) structured over the chain.
 * a is indexed row-major, a[i*d + j] = A[i][j], like every matrix of this ABI: a_mean0 / a_init_mean [d][d],
 * a_cov0 / a_init_cov [d*d][d*d] (SPD), the prior and E[a], cov(a) of the initial q(a), shared by every chain.  Each
 * noise is known or learned as for rxg_lgssm_vmp_noise_f32; both known is allowed (A alone is learned).  One iteration:
 * q(x) under (E[A], E[w_p], E[w_q]) with the factor exp(-1/2 x' Xi x), Xi = E[(A - E[A])' E[w_p] (A - E[A])], on the
 * source state of every transition; then q(a) (with the E[w_p] of that q(x)), q(w_p) (with the new q(a)) and q(w_q).
 * Outputs a_mean[iterations][d][d][batch] and a_cov[iterations][d*d][d*d][batch] (after EVERY iteration), the noise
 * outputs and free_energy as rxg_lgssm_vmp_noise_f32 (the Bethe free energy gains KL(q(a) || prior)).  d in 1..4, m in
 * 1..6, device data, else RXG_ERR_UNSUPPORTED, as are the flags rxg_lgssm_vmp_noise_f32 refuses; a non-SPD a_cov0 /
 * a_init_cov, a missing a_mean / a_cov and every argument rxg_lgssm_vmp_noise_f32 refuses except two known noises give
 * RXG_ERR_BAD_ARG.  status[b] flags a non-positive pivot (also of Xi and of the precision of q(a)).              */
int rxg_lgssm_vmp_transition_f32(rxg_ctx*, int d, int m, int T, int64_t batch, int iterations, const float* a_mean0,
                                 const float* a_cov0, const float* a_init_mean, const float* a_init_cov, const float* B,
                                 const float* m0, const float* S0, const float* u, const float* P, float nu_p0,
                                 const float* inv_scale_p0, const float* init_E_Wp, const float* Q, float nu_q0,
                                 const float* inv_scale_q0, const float* init_E_Wq, const float* y, const uint8_t* ymask,
                                 float* post_mean, float* post_cov, float* a_mean, float* a_cov, float* df_p,
                                 float* inv_scale_p, float* df_q, float* inv_scale_q, double* free_energy, int32_t* status,
                                 unsigned flags);
/* Hierarchical Gaussian Filter, streaming, `iters` VMP iterations per datum
 * [ref: test/models/statespace/hgf_tests.jl:10-69; loop src/inference/streaming.jl:349-407].
 * y[T][batch]; init = (m_z, v_z, m_x, v_x); out[T][4][batch] = (m_x, v_x, m_z, v_z).            */
int rxg_hgf_filter_f32(rxg_ctx*, int T, int64_t batch, int iters, float kappa, float omega,
                       float z_variance, float y_variance, const float init[4], const float* y,
                       float* out, unsigned flags);

/* Same filter with the streaming carry and the Bethe free energy as optional arguments: `init` (first chunk) or
 * `prev[4][batch]` (out[Tc-1] of the previous chunk), exactly one of them non-NULL; free_energy[T][iters][batch] or
 * NULL = the Bethe free energy of each datum's graph after every VMP iteration [ref: definition
 * src/model/plugins/reactivemp_free_energy.jl:84-126; the reference's regression pin for this model is the average
 * over the data after the last iteration, test/models/statespace/hgf_tests.jl:112-119 (1.009879989585)].        */
int rxg_hgf_filter_fe_f32(rxg_ctx*, int T, int64_t batch, int iters, float kappa, float omega,
                          float z_variance, float y_variance, const float init[4], const float* prev,
                          const float* y, float* out, float* free_energy, unsigned flags);
/* Hierarchical Gaussian Filter with the coupling kappa and the volatility offset omega LEARNED per series: mean-field VMP
 * over whole series, `batch` independent chains, all iterations in one launch
 * [ref: model `hgf_1`, test/inference/inference_tests.jl:609-642 (MeanField(), free_energy = true, initialisation
 *  :624-629); GCV rules and average energy :547-607, variance exp(kappa z + omega)]:
 *   omega ~ N(prior[2], prior[3]), kappa ~ N(prior[0], prior[1]), x_0 ~ N(prior[4], prior[5]), z[1] ~ N(prior[6], prior[7]),
 *   z[t] ~ N(z[t-1], precision z_precision) (t >= 2), x[t] ~ GCV(x[t-1], z[t], kappa, omega), y[t] ~ N(x[t], y_variance),
 *   q(kappa) q(omega) q(x_0) prod q(x[t]) q(z[t]).  prior (HOST, 8 floats: mean, variance of kappa, omega, x_0, z[1]);
 *   init (HOST, 8 floats: mean, variance of the initial q(kappa), q(omega), q(z[t]), q(x[t]), the last two for every t).
 *   y[T][batch], NaN = missing step.  Outputs: xz[T][4][batch] = (m_x, v_x, m_z, v_z) of the last iteration (KeepLast),
 *   kw[2][2][batch] = (mean, variance) of q(kappa), then of q(omega); optional (NULL = not wanted): x0[2][batch] = q(x_0),
 *   hist_kw[iterations][2][2][batch] (KeepEach of q(kappa), q(omega)), free_energy[iterations][batch] (fp64, the
 *   mean-field VMP free energy after every iteration), status[batch] (RXG_ERR_NAN for a chain whose update met a
 *   non-finite value).  Products with the GCV node's ExponentialLinearQuadratic messages are GH-31 moment matching
 *   (DESIGN.md section 3.19).  T, batch, iterations >= 1, positive finite variances and z_precision, finite means,
 *   else RXG_ERR_BAD_ARG.  Device pointers (RXG_ERR_UNSUPPORTED otherwise).                                        */
int rxg_hgf_vmp_learn_f32(rxg_ctx*, int T, int64_t batch, int iterations, const float prior[8], float z_precision,
                          float y_variance, const float init[8], const float* y, float* x0, float* xz, float* kw,
                          float* hist_kw, double* free_energy, int32_t* status, unsigned flags);

/* ------------------------------------------------------------------ streaming engine ----------
 * The reference's second entry point: infer(..., autoupdates = ..., keephistory = ...) builds an
 * RxInferenceEngine that re-triggers a ONE-step graph per datum and feeds q(x_t) back as the next
 * prior [ref: executor src/inference/streaming.jl:344-430; @autoupdates x_min_t_mean, x_min_t_cov =
 * mean_cov(q(x_t)) src/inference/autoupdates.jl:614-659; model ipynb:107-113, run ipynb:199-216].
 * Here the datastream is consumed in time-chunks: one call = one fused filtering sweep over Tc data
 * for all chains, with the autoupdate carry made explicit (no hidden state in the ctx):
 *   prev_mean[d][batch]  (device)  in : means of q(x_{t0-1}) -- for the first chunk the broadcast
 *                                       initialisation; afterwards filt_mean[Tc-1] of the last chunk
 *   carry_cov[d][d]      (HOST)    in : covariance of q(x_{t0-1}) (chain independent for a shared
 *                                       model);  out: covariance of q(x_{t0+Tc-1})
 * Model per datum: x_t ~ N(A x_{t-1} + u, P), y_t ~ N(B x_t, Q) (transition first).  Chunking is
 * exact: any split of the stream gives the same posteriors as one call (up to the fp32 rounding of
 * the carried covariance).  Shared model, no mask; device pointers; always synchronous.
 * RXG_U_SEQ_SHARED / RXG_U_SEQ_CHAIN: u is the chunk's input sequence, Tc rows (u[Tc][d] host or
 * u[Tc][d][batch] device); the chunk model is transition first, so row 0 is used.                 */
int rxg_lgssm_filter_chunk_f32(rxg_ctx*, int d, int m, int Tc, int64_t batch, const float* A,
                               const float* B, const float* P, const float* Q, const float* u,
                               const float* prev_mean, float* carry_cov, const float* y,
                               float* filt_mean, float* filt_cov, float* neg_log_evidence,
                               unsigned flags);
/* HGF datastream in time-chunks: prev[4][batch] = out[Tc-1] of the previous chunk (rows m_x, v_x,
 * m_z, v_z: the @autoupdates of hgf_tests.jl:46-49).  First chunk: rxg_hgf_filter_f32 with init.  */
int rxg_hgf_filter_chunk_f32(rxg_ctx*, int Tc, int64_t batch, int iters, float kappa, float omega,
                             float z_variance, float y_variance, const float* prev, const float* y,
                             float* out, unsigned flags);

/* Streaming mean-field VMP with an unknown observation precision -- the reference's `test_model1`
 * [ref: test/inference/inference_tests.jl:752-775; @autoupdates :772-776; rules of
 * test/models/aliases/aliases_gamma_tests.jl]:  x_t_min ~ N(prior), tau ~ Gamma(prior),
 * x_t ~ N(x_t_min, 1/w), y ~ N(x_t, 1/tau), MeanField(), `iters` iterations per datum, priors autoupdated
 * from q(x_t), q(tau).  init = (m_x, v_x, shape, rate) of the @initialization, or prev[4][batch] = out[Tc-1]
 * of the previous time-chunk (then init may be NULL).  y[T][batch]; out[T][4][batch] = (m_x, v_x, shape, rate)
 * after the last iteration of each datum; free_energy[T][iters][batch] or NULL (Bethe free energy per
 * datum and iteration; the reference asserts its average over data to be non-increasing, :846).       */
int rxg_stream_vmp_gamma_f32(rxg_ctx*, int T, int64_t batch, int iters, float w, const float init[4],
                             const float* prev, const float* y, float* out, float* free_energy,
                             unsigned flags);

/* Diagnostic: D[128][64] = A[128][128] * B[64][128]' on the tensor cores (wgmma tf32, 3xTF32 split,
 * register accumulator), row-major device arrays.  Validates the hand-written wgmma descriptors
 * used by the large-state family; no reference counterpart.                                     */
int rxg_selftest_umma_f32(rxg_ctx*, const float* A, const float* B, float* D, unsigned flags);
/* Same for every operand shape the sweeps issue: D[128][n] = A[128][k] * B[n][k]' with
 * (n, k) in {(64,128), (128,64), (64,64), (64,32), (32,32), (32,16), (16,16)}.                    */
int rxg_selftest_umma_shape_f32(rxg_ctx*, int n, int k, const float* A, const float* B, float* D,
                                unsigned flags);

/* Diagnostic: stream n floats from each of n_read input rows (src[n_read][n]) and store their sum into each of
 * n_write output rows (dst[n_write][n]) -- a dependency-free kernel with a chosen HBM read : write mix, the
 * yardstick for the sweep kernels' achieved bandwidth (bench_extra.py --which stream).  No reference counterpart. */
int rxg_selftest_stream_f32(rxg_ctx*, int64_t n, int n_read, int n_write, const float* src, float* dst,
                            unsigned flags);

/* Diagnostic: write bandwidth (GB/s) of the host-side covariance broadcast into dst[rows][batch] (host memory).      */
double rxg_selftest_host_fill_gbs(float* dst, int64_t rows, int64_t batch, int nthreads, int reps);

/* ------------------------------------------------------------------ multi-GPU ----------------
 * Chains are independent: rank g owns chains [g*batch/G, (g+1)*batch/G); the only collective is
 * the all-gather of posterior marginals at the end (the reference has no distributed path).
 * rxg_comm_unique_id fills a 128-byte NCCL id on rank 0; the host broadcasts it out of band.    */
int rxg_comm_unique_id(void* id128);
int rxg_comm_init(rxg_ctx*, int nranks, int rank, const void* id128);
/* Gather each rank's (mean[T][d][b_local], cov[T][d][d][b_local]) slab into
 * gathered_*[G][...] (rank-major, each slab contiguous).  Device pointers only.
 * With RXG_COV_REPLICATE (shared model on every rank, no ymask: the covariances do not depend on
 * the chain, SURVEY.md appendix A.1) only the means cross NVLink; gathered_cov[G][T][d][d][b_local]
 * is filled locally from post_cov (its first chain column, or the [T][d][d] table when
 * RXG_COV_SHARED_OUT is also set) at HBM write speed, concurrently with the gather.  Results are
 * bit-identical to the full gather.                                                              */
int rxg_allgather_posteriors(rxg_ctx*, int d, int T, int64_t batch_local, const float* post_mean,
                             const float* post_cov, float* gathered_mean, float* gathered_cov,
                             unsigned flags);


/* ------------------------------------------------------------------ peer-mapped gather ---------
 * The all-gather WITHOUT a collective launch: every rank maps its peers' gathered buffers (CUDA IPC over
 * NVLink / NVSwitch) and the fused smoothing sweep stores each smoothed posterior straight into all G
 * buffers while the backward recursion is still running (SURVEY.md section 8e: "issue ... finished time-slabs
 * ... while earlier slabs are still being computed" -- here at the granularity of one time step).
 * Host protocol (one process per GPU; the host exchanges the 64-byte handles out of band, e.g.
 * torch.distributed / MPI / a Julia Distributed channel):
 *   1. rxg_device_alloc the gathered buffers [G][T][d][b_local] (+ [G][T][d][d][b_local]) and one flag
 *      buffer of RXG_MAX_PEERS ints (zero it with rxg_device_memset);
 *   2. rxg_peer_export each, all-gather the handles, rxg_peer_open the G-1 remote ones;
 *   3. rxg_peer_group(nranks, rank, flag pointers as mapped here);
 *   4. rxg_lgssm_smooth_gather_f32 (or any compute + rxg_peer_allgather_f32) per step.
 * Ranks inside ONE process (several contexts) skip step 2's export/open and pass plain device pointers.   */
int rxg_device_alloc(rxg_ctx*, size_t bytes, void** dev_ptr);
int rxg_device_free(rxg_ctx*, void* dev_ptr);
int rxg_device_memset(rxg_ctx*, void* dev_ptr, int value, size_t bytes);
/* synchronous copies on the ctx stream -- for hosts without a CUDA binding of their own (the Julia shim, C hosts)  */
int rxg_memcpy_h2d(rxg_ctx*, void* dst_dev, const void* src_host, size_t bytes);
int rxg_memcpy_d2h(rxg_ctx*, void* dst_host, const void* src_dev, size_t bytes);
int rxg_peer_export(rxg_ctx*, const void* dev_ptr, void* handle64);
int rxg_peer_open(rxg_ctx*, const void* handle64, void** dev_ptr);
int rxg_peer_close(rxg_ctx*, void* dev_ptr);
/* flag_ptrs[g] = rank g's flag buffer as mapped in this process (own buffer for g == rank); nranks <= RXG_MAX_PEERS */
int rxg_peer_group(rxg_ctx*, int nranks, int rank, void* const* flag_ptrs);
/* device-side barrier over the group on the ctx stream (st.release.sys / ld.acquire.sys on the flags)     */
int rxg_peer_barrier(rxg_ctx*, unsigned flags);
/* generic all-gather of any posterior array (HGF outputs, filtered means, ...): `local` (n_local floats, may
 * already be the own slab gathered[rank] + rank * n_local) is stored into slab `rank` of every gathered[g],
 * then the barrier.  On completion gathered[rank] holds all G slabs.                                       */
int rxg_peer_allgather_f32(rxg_ctx*, int64_t n_local, const float* local, float* const* gathered, unsigned flags);
/* rxg_lgssm_smooth_f32 + the all-gather of its posteriors in one call: gathered_mean[g] / gathered_cov[g] are the
 * bases of rank g's [G][T][d][b_local] / [G][T][d][d][b_local] buffers as mapped here.  Shared-model gain-table
 * path: the sweep kernel itself stores to the peers (no second pass); other paths push their finished slab.
 * RXG_COV_REPLICATE (shared model, no mask): only the means cross NVLink, the other ranks' covariance slabs are
 * replicated locally from the [T][d][d] table concurrently with the sweep (gathered_cov[g != rank] may be NULL);
 * the buffers end up bit-identical to the full gather.  neg_log_evidence / status are local ([b_local]).
 * A caller must not start the next gather into the same buffers before every rank has consumed the result.
 * RXG_U_SEQ_SHARED / RXG_U_SEQ_CHAIN are refused with RXG_ERR_UNSUPPORTED before anything runs.              */
int rxg_lgssm_smooth_gather_f32(rxg_ctx*, int d, int m, int T, int64_t batch_local, const float* A,
                                const float* B, const float* P, const float* Q, const float* m0,
                                const float* S0, const float* u, const float* y, const uint8_t* ymask,
                                float* const* gathered_mean, float* const* gathered_cov,
                                float* neg_log_evidence, int32_t* status, unsigned flags);

/* ------------------------------------------------------------------ Delta node (nonlinear maps) ----------
 * z := f(x) between Gaussian nodes with meta Linearization() or Unscented(alpha, beta, kappa)
 * [ref: docs/src/manuals/inference/delta-node.md; paper/example.jl].  The user supplies CUDA C++ source defining
 *   template <class S> __device__ void f(const S* x, S* z);   (transition, R^d -> R^d)
 *   template <class S> __device__ void g(const S* x, S* y);   (optional observation map, R^d -> R^m)
 * calling math functions unqualified (sin, cos, tan, exp, log, sqrt, tanh, atan, atan2, pow, fabs).  The library
 * compiles it at run time with NVRTC, loaded with dlopen once per process by the first compile: the path in
 * RXG_NVRTC as rxg_create read it for the context that compiles first, else libnvrtc.so.12 (rxg_delta_check_source
 * always uses the soname); later overrides are ignored once NVRTC is loaded.  The source is compiled
 * with the library's Delta header, for sm_90a and exactly one (d, m), d and m in 1..8.  Linearization runs in fp32
 * (Jacobians by forward-mode dual numbers); Unscented in fp64 (2d + 1 sigma points; ut = {alpha, beta, kappa} or
 * NULL for ReactiveMP's Unscented() defaults {1e-3, 2, 0}).  Without NVRTC the entries return RXG_ERR_UNSUPPORTED;
 * a compile error returns RXG_ERR_BAD_ARG with the compiler log in `log` (and in rxg_last_error).
 * A model belongs to its context: the context caches one module per (source, names, d, m, method, ut), so a second
 * create of the same model compiles nothing, and rxg_destroy unloads them all.
 * Model constants (row-major host arrays) are shared by every chain; data are device arrays (RXG_PTR_DEVICE is
 * required).  Per-chain status: RXG_ERR_NOT_SPD (a predicted or innovation covariance is not SPD), RXG_ERR_NAN.  */
typedef struct rxg_delta_model rxg_delta_model;
#define RXG_DELTA_LINEARIZATION 0
#define RXG_DELTA_UNSCENTED 1
/* Compile check without a context or a GPU: RXG_OK, or RXG_ERR_BAD_ARG with the NVRTC log (which also carries the
 * ptxas register / spill report of both kernels on success).                                                       */
int rxg_delta_check_source(const char* source, const char* f_name, const char* g_name, int d, int m, int method,
                           const double ut[3], char* log, size_t log_cap);
int rxg_delta_model_create(rxg_ctx*, const char* source, const char* f_name, const char* g_name, int d, int m,
                           int method, const double ut[3], rxg_delta_model** out, char* log, size_t log_cap);
/* NVRTC compilations this context has run (a cached create adds none)                                             */
long long rxg_delta_compile_count(const rxg_ctx*);
/* Whole series, one fused launch: x[1] ~ N(m0, S0), x[t] = f(x[t-1]) + N(0, P), y[t] ~ N(B x[t], Q) (g NULL) or
 * N(g(x[t]), Q) (B may be NULL); the EKF / UKF forward pass then the ERTS / URTS backward pass, the transition
 * linearised at the filtered marginals.  y[T][m][batch]; ymask[T][batch] (1 = observed) or NULL;
 * post_mean[T][d][batch], post_cov[T][d][d][batch]; filt_mean / filt_cov (same shapes) or NULL; status[batch] or NULL. */
int rxg_delta_smooth_f32(rxg_ctx*, const rxg_delta_model* model, int T, int64_t batch, const float* m0,
                         const float* S0, const float* P, const float* B, const float* Q, const float* y,
                         const uint8_t* ymask, float* post_mean, float* post_cov, float* filt_mean, float* filt_cov,
                         int32_t* status, unsigned flags);
/* Streaming filter, one time-chunk of Tc data.  Carry q(x) = carry_mean[d][batch], carry_cov[d][d][batch] (device,
 * updated in place); every datum pushes it through f (+ P) and then updates it by y.  Known noise: Q (carry_tau and
 * filt_tau NULL).  Learned precision (m = 1, B the observation row, no g, Q NULL): y ~ N(B x, 1/tau), q(x) q(tau),
 * carry_tau[2][batch] = (shape, rate) of q(tau), which is both the next datum's Gamma prior and its initial q(tau),
 * and `iters` VMP iterations per datum; filt_tau[Tc][2][batch] or NULL.  filt_mean[Tc][d][batch] /
 * filt_cov[Tc][d][d][batch] or NULL.  The carry is rounded to fp32 after every datum, so splitting a stream into
 * chunks gives the same result, bit for bit, as one call.                                                           */
int rxg_delta_filter_chunk_f32(rxg_ctx*, const rxg_delta_model* model, int Tc, int64_t batch, const float* P,
                               const float* B, const float* Q, int iters, const float* y, const uint8_t* ymask,
                               float* carry_mean, float* carry_cov, float* carry_tau, float* filt_mean, float* filt_cov,
                               float* filt_tau, int32_t* status, unsigned flags);

#ifdef __cplusplus
}
#endif
#endif /* RXGAUSS_H */
