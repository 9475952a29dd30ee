// Test harness (NOT part of librxgauss.so): compiles the body of the learned-kappa/omega HGF kernel
// (csrc/rxg_hgf_learn.cuh, __host__ __device__) for the host so that the exact code the GPU runs can be checked against
// the fp64 reference without a GPU (tests/test_hgf_learn.py).  The product path has no CPU route: rxg_hgf_vmp_learn_f32
// launches the CUDA kernel or fails.  gh_t / gh_lw2 are the 31 Gauss-Hermite nodes and log2 weights the C entry uploads.
#include <cuda_runtime.h>
#include "../../rxinfer.jl_b200/csrc/rxg_hgf_learn.cuh"

extern "C" int hgf_learn_host_run(int T, long long batch, int iters, const float* prior, float z_precision,
                                  float y_variance, const float* init, const float* gh_t, const float* gh_lw2,
                                  const float* y, float* x0, float* xz, float* kw, float* hist_kw, double* fe,
                                  int* status) {
    using namespace rxg::hgfl;
    GH gh;
    for (int i = 0; i < NGH; ++i) { gh.t[i] = gh_t[i]; gh.lw2[i] = gh_lw2[i]; }
    fill_vfix(gh);
    const Prm p{prior[0], prior[1], prior[2], prior[3], prior[4], prior[5], prior[6], prior[7], z_precision, y_variance,
                init[0], init[1], init[2], init[3], init[4], init[5], init[6], init[7]};
    const Args a{T, iters, batch, p, y, x0, xz, kw, hist_kw, fe};
    for (long long b = 0; b < batch; ++b) status[b] = fe ? chain<true>(b, a, gh) : chain<false>(b, a, gh);
    return 0;
}
