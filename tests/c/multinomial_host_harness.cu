// Test harness (NOT part of librxgauss.so): compiles the per-chain bodies of the multinomial regression kernels
// (csrc/rxg_multinomial.cuh, __host__ __device__) for the host, with one "lane" owning every column, so that the code the
// GPU runs can be checked against the fp64 reference without a GPU (tests/test_multinomial.py).  The product path has no
// CPU route: the rxg_multinomial_polya_* entries launch CUDA kernels or fail.  The prior block is what the C entries
// derive from xi0 and W0: m0 = W0^-1 xi0 [D], then S0 = W0^-1 [D][D].
#include <cuda_runtime.h>

#include <vector>

#include "../../rxinfer.jl_b200/csrc/rxg_multinomial.cuh"

using namespace rxg::mnp;

static std::vector<double> log_fact_table() {
    std::vector<double> lf(LF_N);
    for (int i = 0; i < LF_N; ++i) lf[i] = lgamma(i + 1.0);
    return lf;
}

struct Arrays {
    std::vector<double> S, m, d, u, r, S2, m2;
    explicit Arrays(int D) : S(D * D), m(D), d(D), u(D), r(D), S2(D * D), m2(D) {}
    Work a() { return Work{S.data(), m.data(), d.data(), u.data(), r.data()}; }
    Work b() { return Work{S2.data(), m2.data(), d.data(), u.data(), r.data()}; }
};

// whole data sets: y[n][K][batch]; outputs as rxg_multinomial_polya_vmp_f32
extern "C" int multinomial_host_vmp(int K, int n, long long batch, int iters, const double* prior, const int* y,
                                    float* mean, float* cov, double* fe, float* hist_mean, float* hist_cov, int* status) {
    if (K < 2 || K > MAX_K) return -1;
    const int D = K - 1;
    const std::vector<double> lf = log_fact_table();
    const Out o{batch, mean, cov, hist_mean, hist_cov, fe};
    for (long long c = 0; c < batch; ++c) {
        double Y[MAX_K] = {}, lcoef = 0.0;
        bool bad = false;
        for (int i = 0; i < n; ++i) {
            int32_t v[MAX_K] = {};
            for (int k = 0; k < K; ++k) v[k] = y[((long long)i * K + k) * batch + c];
            if (!add_sample<MAX_K>(K, v, lf.data(), Y, lcoef)) bad = true;
        }
        const double lc = suffix_totals<MAX_K>(K, Y, lcoef);
        std::vector<double> b(D), nn(D);
        for (int k = 0; k < D; ++k) {
            b[k] = (Y[k] - Y[k + 1]) - 0.5 * Y[k];
            nn[k] = Y[k];
        }
        Arrays ar(D);
        int st = bad ? ST_BAD : 0;
        offline(0, 1, D, iters, prior, prior + D, b.data(), nn.data(), lc, ar.a(), o, c, st);
        status[c] = st;
    }
    return 0;
}

// online: y[T][K][batch]; carry m[D][batch], S[D][D][batch] updated in place (prior block when `start` is set)
extern "C" int multinomial_host_online(int K, int T, long long batch, int iters, const double* prior, int start,
                                       double* m_carry, double* S_carry, const int* y, float* hist_mean, float* hist_cov,
                                       double* fe, int* status) {
    if (K < 2 || K > MAX_K) return -1;
    const int D = K - 1;
    const std::vector<double> lf = log_fact_table();
    const Out o{batch, nullptr, nullptr, hist_mean, hist_cov, fe};
    for (long long c = 0; c < batch; ++c) {
        Arrays ar(D);
        Work base = ar.a(), w = ar.b();
        for (int j = 0; j < D; ++j) {
            base.m[j] = start ? prior[j] : m_carry[j * batch + c];
            for (int i = 0; i < D; ++i) base.S[i * D + j] = start ? prior[D + i * D + j] : S_carry[((long long)i * D + j) * batch + c];
        }
        std::vector<double> b(D), nn(D);
        int32_t cnt[MAX_K];
        int st = 0;
        online<MAX_K>(0, 1, K, T, iters, y, c, lf.data(), base, w, cnt, b.data(), nn.data(), o, st);
        for (int j = 0; j < D; ++j) {
            m_carry[j * batch + c] = base.m[j];
            for (int i = 0; i < D; ++i) S_carry[((long long)i * D + j) * batch + c] = base.S[i * D + j];
        }
        status[c] = st;
    }
    return 0;
}
