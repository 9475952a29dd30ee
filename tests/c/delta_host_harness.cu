// Test harness (NOT part of librxgauss.so): compiles the Delta-node header (csrc/rxg_delta.cuh, __host__ __device__) for
// the host, so that its dual numbers and the exact chain steps the NVRTC-compiled kernels run can be checked against
// analytic Jacobians and the fp64 oracle without a GPU (tests/test_delta.py).
#include <math.h>

#include "../../rxinfer.jl_b200/csrc/rxg_delta.cuh"

// z[k] = the k-th overload applied to (x0, x1); its analytic Jacobian lives in tests/test_delta.py (DUAL_OPS)
struct AllOps {
    template <class S> static __host__ __device__ void eval(const S* x, S* z) {
        const S a = x[0], b = x[1];
        z[0] = sin(a); z[1] = cos(a); z[2] = tan(a); z[3] = exp(a); z[4] = log(a); z[5] = sqrt(a); z[6] = tanh(a);
        z[7] = atan(a); z[8] = fabs(b); z[9] = atan2(a, b); z[10] = atan2(a, 2.0); z[11] = atan2(1.5, b);
        z[12] = pow(a, 2.5); z[13] = pow(a, b); z[14] = pow(1.7, b); z[15] = -a * b + a / b - 2.0 / b + 3 * a - 0.5;
    }
};
enum { N_OPS = 16 };

extern "C" int delta_host_dual_ops(const float* x, float* val, float* jac) {
    rxgd::Dual<2> xd[2], z[N_OPS];
    for (int i = 0; i < 2; ++i) { xd[i] = rxgd::Dual<2>(x[i]); xd[i].g[i] = 1.f; }
    AllOps::eval(xd, z);
    for (int k = 0; k < N_OPS; ++k) {
        val[k] = z[k].v;
        jac[2 * k] = z[k].g[0]; jac[2 * k + 1] = z[k].g[1];
    }
    return N_OPS;
}

// the test transition of every d: z_i = 0.9 x_i + 0.2 sin(x_{i+1 mod d}); observation y = B x (m = 1)
template <int DD> struct WaveD {
    template <class S> static __host__ __device__ void eval(const S* x, S* z) {
        for (int i = 0; i < DD; ++i) z[i] = 0.9 * x[i] + 0.2 * sin(x[(i + 1) % DD]);
    }
};
struct NoG {
    template <class S> static __host__ __device__ void eval(const S*, S*) {}
};
template <int DD, int METH> struct Cfg {
    enum { D = DD, M = 1, METHOD = METH, HAS_G = 0 };
    static constexpr double ALPHA = 1e-3, BETA = 2.0, KAPPA = 0.0;
    typedef WaveD<DD> F;
    typedef NoG G;
};

static void pack(rxgd::Params& p, int d, const float* m0, const float* S0, const float* P, const float* B, const float* Q) {
    for (int i = 0; i < d; ++i) p.m0[i] = m0 ? m0[i] : 0.f;
    for (int i = 0; i < d * d; ++i) { p.S0[i] = S0 ? S0[i] : 0.f; p.P[i] = P[i]; }
    for (int i = 0; i < d; ++i) p.B[i] = B[i];
    p.Q[0] = Q ? Q[0] : 0.f;
}

// one chain (batch 1): the smoother (y[T], mean[T][d], cov[T][d][d]) and the streaming VMP of the learned precision
extern "C" int delta_host_smooth(int d, int method, int T, const float* m0, const float* S0, const float* P, const float* B,
                                 const float* Q, const float* y, const unsigned char* mask, float* mean, float* cov) {
    rxgd::Params p;
    pack(p, d, m0, S0, P, B, Q);
    int st = -1;
#define CASE(DD)                                                                                                     \
    case DD:                                                                                                         \
        if (method) rxgd::smooth_chain<Cfg<DD, 1>>(p, T, 1, 0, y, mask, mean, cov, nullptr, nullptr, &st);          \
        else rxgd::smooth_chain<Cfg<DD, 0>>(p, T, 1, 0, y, mask, mean, cov, nullptr, nullptr, &st);                 \
        break;
    switch (d) { CASE(1) CASE(2) CASE(4) CASE(8) default: return -1; }
#undef CASE
    return st;
}

extern "C" int delta_host_vmp(int d, int method, int T, int iters, const float* P, const float* c, const float* y,
                              float* carry_mean, float* carry_cov, float* carry_tau, float* mean, float* cov, float* tau) {
    rxgd::Params p;
    pack(p, d, nullptr, nullptr, P, c, nullptr);
    int st = -1;
#define CASE(DD)                                                                                                          \
    case DD:                                                                                                              \
        if (method) rxgd::filter_chain<Cfg<DD, 1>>(p, T, 1, 0, y, nullptr, carry_mean, carry_cov, carry_tau, iters, mean, \
                                                   cov, tau, &st);                                                        \
        else rxgd::filter_chain<Cfg<DD, 0>>(p, T, 1, 0, y, nullptr, carry_mean, carry_cov, carry_tau, iters, mean, cov,   \
                                            tau, &st);                                                                    \
        break;
    switch (d) { CASE(1) CASE(2) CASE(4) CASE(8) default: return -1; }
#undef CASE
    return st;
}
