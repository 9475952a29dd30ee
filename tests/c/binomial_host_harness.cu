// Test harness (NOT part of librxgauss.so): compiles the per-chain body of the binomial regression kernel
// (csrc/rxg_polya.cuh, __host__ __device__) for the host so that the code the GPU runs can be checked against the fp64
// reference without a GPU (tests/test_binomial.py).  The product path has no CPU route: rxg_binomial_polya_vmp_f32
// launches a CUDA kernel or fails.  The prior block is what the C entry derives from xi0 and W0: xi0[p], W0[p][p],
// m0[p], S0[p][p], log|W0|, xi0' m0.
#include <cuda_runtime.h>
#include "../../rxinfer.jl_b200/csrc/rxg_polya.cuh"

extern "C" int binomial_host_run(int p, int N, long long batch, int iters, const double* xi0, const double* W0,
                                 const double* m0, const double* S0, double logdetW0, double quad0, const float* X,
                                 const int* y, const int* n, float* mean, float* cov, double* fe, float* hist_mean,
                                 float* hist_cov, int* status) {
    using namespace rxg::polya;
    Prior pr{};
    for (int i = 0; i < p; ++i) {
        pr.xi0[i] = xi0[i];
        pr.m0[i] = m0[i];
        for (int j = 0; j < p; ++j) {
            pr.W0[i * MAX_P + j] = W0[i * p + j];
            pr.S0[i * MAX_P + j] = S0[i * p + j];
        }
    }
    pr.logdetW0 = logdetW0;
    pr.quad0 = quad0;
    const Args a{N, iters, batch, X, y, n, mean, cov, fe, hist_mean, hist_cov};
    for (long long b = 0; b < batch; ++b) {
        int st;
        switch (p) {
#define CASE(PP) case PP: st = chain<PP>(b, a, pr); break;
            CASE(1) CASE(2) CASE(3) CASE(4) CASE(5) CASE(6) CASE(7) CASE(8)
#undef CASE
            default: return -1;
        }
        status[b] = st;
    }
    return 0;
}

extern "C" int binomial_select_path(long long batch, int N, int p, int sm_count) {
    return rxg::polya::select_path(batch, N, p, sm_count);
}
extern "C" int binomial_group_chains_per_sm() { return (int)rxg::polya::GROUP_CHAINS_PER_SM; }
extern "C" int binomial_group_min_n() { return rxg::polya::GROUP_MIN_N; }
