// Test harness (NOT part of librxgauss.so): compiles the body of the HMM kernel (csrc/rxg_hmm.cuh, __host__ __device__)
// for the host so that the exact code the GPU runs can be checked against the fp64 reference without a GPU
// (tests/test_hmm.py).  The product path has no CPU route: rxg_hmm_vmp_f32 launches the CUDA kernel or fails.
// prm is the fp64 constant block the C entry uploads (rxg::hmm::off_*); learn_A / learn_B select learned or known matrices.
#include <vector>

#include <cuda_runtime.h>
#include "../../rxinfer.jl_b200/csrc/rxg_hmm.cuh"

extern "C" int hmm_host_run(int K, int M, int T, long long batch, int iters, int learn_A, int learn_B, const double* prm,
                            const unsigned char* x, float* s_prob, float* s0_prob, float* A_alpha, float* B_alpha,
                            double* fe, float* hist_s, float* hist_A, float* hist_B, int* status) {
    rxg::hmm::Args a{T, M, iters, batch, learn_A, learn_B, prm, x, s_prob, s0_prob, A_alpha, B_alpha, fe, hist_s, hist_A,
                     hist_B};
    std::vector<float> fsh(M * K);
    std::vector<double> dsh(K * K + M * K);
    for (long long b = 0; b < batch; ++b) {
        int st;
        switch (K) {
#define CASE(KK) case KK: st = rxg::hmm::chain<KK>(b, a, fsh.data(), dsh.data(), 1); break;
            CASE(2) CASE(3) CASE(4) CASE(5) CASE(6) CASE(7) CASE(8)
#undef CASE
            default: return -1;
        }
        status[b] = st;
    }
    return 0;
}
