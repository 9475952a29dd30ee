// Test harness (NOT part of librxgauss.so): compiles the body of the Gaussian-emission HMM kernel (csrc/rxg_hmm_gauss.cuh,
// __host__ __device__) for the host so that the exact code the GPU runs can be checked against the fp64 reference without a
// GPU (tests/test_hmm_gauss.py).  The product path has no CPU route: rxg_hmm_gauss_vmp_f32 launches the CUDA kernel or
// fails.  prm is the fp64 constant block the C entry uploads (rxg::hmmg::off_states, layout); learn_A selects q(A) or a
// known A.
#include <vector>

#include <cuda_runtime.h>
#include "../../rxinfer.jl_b200/csrc/rxg_hmm_gauss.cuh"

extern "C" int hmm_gauss_host_run(int d, int K, int T, long long batch, int iters, int learn_A, const double* prm,
                                  const float* y, float* s_prob, float* s0_prob, float* A_alpha, float* m_mean, float* m_cov,
                                  float* w_df, float* w_inv_scale, double* fe, float* hist_s, float* hist_A,
                                  float* hist_m_mean, float* hist_m_cov, float* hist_w_df, float* hist_w_inv_scale,
                                  int* status) {
    using namespace rxg::hmmg;
    Args a{T, iters, batch, learn_A, prm, y, s_prob, s0_prob, A_alpha, m_mean, m_cov, w_df, w_inv_scale, fe, hist_s,
           hist_A, hist_m_mean, hist_m_cov, hist_w_df, hist_w_inv_scale};
    std::vector<float> fsh(f_slots(d, K));
    std::vector<double> dsh(K * K + K * acc_slots(d));
    for (long long b = 0; b < batch; ++b) {
        int st;
        switch (d * 16 + K) {
#define CASE(DD, KK) case DD * 16 + KK: st = chain<DD, KK>(b, a, fsh.data(), dsh.data(), 1); break;
#define DCASES(DD) CASE(DD, 2) CASE(DD, 3) CASE(DD, 4) CASE(DD, 5) CASE(DD, 6) CASE(DD, 7) CASE(DD, 8)
            DCASES(1) DCASES(2) DCASES(3) DCASES(4)
#undef DCASES
#undef CASE
            default: return -1;
        }
        status[b] = st;
    }
    return 0;
}
