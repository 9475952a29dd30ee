// Test harness (NOT part of librxgauss.so): compiles the per-chain body of the Gamma mixture kernel
// (csrc/rxg_gamma_mixture.cuh, __host__ __device__) for the host so that the code the GPU runs can be checked against the
// fp64 reference without a GPU (tests/test_gamma_mixture.py).  The product path has no CPU route:
// rxg_gamma_mixture_vmp_f32 launches a CUDA kernel or fails.  prm is the fp64 constant block the C entry builds.
#include <cuda_runtime.h>
#include <vector>
#include "../../rxinfer.jl_b200/csrc/rxg_gamma_mixture.cuh"

extern "C" int gamma_mixture_host_run(int K, int N, long long batch, int iters, const double* prm, const float* y,
                                      float* alpha, float* a_hat, float* b_shape, float* b_rate, double* fe, float* z_prob,
                                      float* hist_a, float* hist_b_shape, float* hist_b_rate, int* status) {
    using namespace rxg::gamix;
    const Args a{K, N, iters, batch, prm, y, alpha, a_hat, b_shape, b_rate, fe, z_prob, hist_a, hist_b_shape, hist_b_rate};
    std::vector<double> st(N_SLOTS * MAX_K);
    for (long long b = 0; b < batch; ++b) {
        switch (K) {
#define CASE(KK) case KK: status[b] = chain<KK>(b, a, st.data(), 1); break;
            CASE(2) CASE(3) CASE(4) CASE(5) CASE(6) CASE(7) CASE(8)
#undef CASE
            default: return -1;
        }
    }
    return 0;
}

extern "C" int gamma_mixture_point_mass_shape(double ash, double art, double n, double c, double a0, double* a) {
    return rxg::gamix::point_mass_shape(ash, art, n, c, a0, *a) ? 1 : 0;
}

extern "C" double gamma_mixture_trigamma(double x) { return rxg::gamix::trigamma(x); }
