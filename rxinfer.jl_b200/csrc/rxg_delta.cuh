// Delta node (z := h(x)) between Gaussian nodes: the Linearization and Unscented moment approximations of a user
// function, the EKF / UKF forward step, the ERTS / URTS backward step and the per-datum VMP step of a Delta
// transition observed with a Gamma-learned precision.
//
// This header has no #includes: the library embeds it as a string and compiles it at run time with NVRTC,
// together with the user's CUDA source and a generated instantiation tail (rxg_delta.cu).  Every body is
// __host__ __device__, so a host harness can compile it too (tests/c/delta_host_harness.cu); such a harness
// includes <math.h> first.
//
// User contract: `template <class S> __device__ void f(const S* x, S* z)` (and optionally g), calling math
// functions unqualified.  S is Dual<D> (Linearization: value and Jacobian in fp32, forward mode) or double
// (Unscented: sigma points in fp64).  Argument-dependent lookup finds the Dual overloads below.
#ifndef RXGD_HD
#define RXGD_HD __host__ __device__ __forceinline__
#endif

namespace rxgd {

enum { OK = 0, ERR_NOT_SPD = 4, ERR_NAN = 5 };     // the RXG_ERR_* codes of include/rxgauss.h
enum { LINEARIZATION = 0, UNSCENTED = 1 };

// ------------------------------------------------------------------ dual numbers (forward mode, N tangents)
template <int N>
struct Dual {
    float v;
    float g[N];
    RXGD_HD Dual() : v(0.f) { for (int i = 0; i < N; ++i) g[i] = 0.f; }
    RXGD_HD Dual(float x) : v(x) { for (int i = 0; i < N; ++i) g[i] = 0.f; }
    RXGD_HD Dual(double x) : v((float)x) { for (int i = 0; i < N; ++i) g[i] = 0.f; }
    RXGD_HD Dual(int x) : v((float)x) { for (int i = 0; i < N; ++i) g[i] = 0.f; }

    // r = (value, s * a.g) -- the chain rule of a unary function with derivative s
    RXGD_HD static Dual chain(float value, float s, const Dual& a) {
        Dual r; r.v = value;
        for (int i = 0; i < N; ++i) r.g[i] = s * a.g[i];
        return r;
    }
    // r = (value, sa * a.g + sb * b.g)
    RXGD_HD static Dual chain2(float value, float sa, const Dual& a, float sb, const Dual& b) {
        Dual r; r.v = value;
        for (int i = 0; i < N; ++i) r.g[i] = sa * a.g[i] + sb * b.g[i];
        return r;
    }

    friend RXGD_HD Dual operator-(const Dual& a) { return chain(-a.v, -1.f, a); }
    friend RXGD_HD Dual operator+(const Dual& a) { return a; }
    friend RXGD_HD Dual operator+(const Dual& a, const Dual& b) { return chain2(a.v + b.v, 1.f, a, 1.f, b); }
    friend RXGD_HD Dual operator-(const Dual& a, const Dual& b) { return chain2(a.v - b.v, 1.f, a, -1.f, b); }
    friend RXGD_HD Dual operator*(const Dual& a, const Dual& b) { return chain2(a.v * b.v, b.v, a, a.v, b); }
    friend RXGD_HD Dual operator/(const Dual& a, const Dual& b) {
        const float q = a.v / b.v;
        return chain2(q, 1.f / b.v, a, -q / b.v, b);
    }
    friend RXGD_HD Dual operator+(const Dual& a, double c) { return chain(a.v + (float)c, 1.f, a); }
    friend RXGD_HD Dual operator+(double c, const Dual& a) { return chain((float)c + a.v, 1.f, a); }
    friend RXGD_HD Dual operator-(const Dual& a, double c) { return chain(a.v - (float)c, 1.f, a); }
    friend RXGD_HD Dual operator-(double c, const Dual& a) { return chain((float)c - a.v, -1.f, a); }
    friend RXGD_HD Dual operator*(const Dual& a, double c) { return chain(a.v * (float)c, (float)c, a); }
    friend RXGD_HD Dual operator*(double c, const Dual& a) { return chain((float)c * a.v, (float)c, a); }
    friend RXGD_HD Dual operator/(const Dual& a, double c) { return chain(a.v / (float)c, 1.f / (float)c, a); }
    friend RXGD_HD Dual operator/(double c, const Dual& a) {
        const float q = (float)c / a.v;
        return chain(q, -q / a.v, a);
    }
    RXGD_HD Dual& operator+=(const Dual& b) { return *this = *this + b; }
    RXGD_HD Dual& operator-=(const Dual& b) { return *this = *this - b; }
    RXGD_HD Dual& operator*=(const Dual& b) { return *this = *this * b; }
    RXGD_HD Dual& operator/=(const Dual& b) { return *this = *this / b; }
    // comparisons act on the value (branches of a piecewise function follow the linearisation point)
    friend RXGD_HD bool operator<(const Dual& a, const Dual& b) { return a.v < b.v; }
    friend RXGD_HD bool operator>(const Dual& a, const Dual& b) { return a.v > b.v; }
    friend RXGD_HD bool operator<=(const Dual& a, const Dual& b) { return a.v <= b.v; }
    friend RXGD_HD bool operator>=(const Dual& a, const Dual& b) { return a.v >= b.v; }

    friend RXGD_HD Dual sin(const Dual& a) { return chain(sinf(a.v), cosf(a.v), a); }
    friend RXGD_HD Dual cos(const Dual& a) { return chain(cosf(a.v), -sinf(a.v), a); }
    friend RXGD_HD Dual tan(const Dual& a) { const float t = tanf(a.v); return chain(t, 1.f + t * t, a); }
    friend RXGD_HD Dual exp(const Dual& a) { const float e = expf(a.v); return chain(e, e, a); }
    friend RXGD_HD Dual log(const Dual& a) { return chain(logf(a.v), 1.f / a.v, a); }
    friend RXGD_HD Dual sqrt(const Dual& a) { const float s = sqrtf(a.v); return chain(s, 0.5f / s, a); }
    friend RXGD_HD Dual tanh(const Dual& a) { const float t = tanhf(a.v); return chain(t, 1.f - t * t, a); }
    friend RXGD_HD Dual atan(const Dual& a) { return chain(atanf(a.v), 1.f / (1.f + a.v * a.v), a); }
    friend RXGD_HD Dual fabs(const Dual& a) { return chain(fabsf(a.v), a.v < 0.f ? -1.f : 1.f, a); }
    friend RXGD_HD Dual atan2(const Dual& y, const Dual& x) {
        const float r2 = x.v * x.v + y.v * y.v;
        return chain2(atan2f(y.v, x.v), x.v / r2, y, -y.v / r2, x);
    }
    friend RXGD_HD Dual atan2(const Dual& y, double x) { return atan2(y, Dual(x)); }
    friend RXGD_HD Dual atan2(double y, const Dual& x) { return atan2(Dual(y), x); }
    friend RXGD_HD Dual pow(const Dual& a, double c) {
        const float p = powf(a.v, (float)c);
        return chain(p, (float)c * powf(a.v, (float)c - 1.f), a);
    }
    friend RXGD_HD Dual pow(double c, const Dual& b) {
        const float p = powf((float)c, b.v);
        return chain(p, p * logf((float)c), b);
    }
    friend RXGD_HD Dual pow(const Dual& a, const Dual& b) {
        const float p = powf(a.v, b.v);
        return chain2(p, b.v * powf(a.v, b.v - 1.f), a, p * logf(a.v), b);
    }
};

template <int M> struct RealOf { typedef float T; };        // Linearization: fp32
template <> struct RealOf<UNSCENTED> { typedef double T; };  // Unscented: fp64 (see moments_ut)

template <class R> RXGD_HD bool is_finite(R x) { return x == x && x - x == R(0); }

// ------------------------------------------------------------------ small dense algebra (row-major, compile-time sizes)
// lower Cholesky factor of the symmetric part of A; false if a pivot is not positive or not finite
template <int N, class R>
RXGD_HD bool cholesky(const R* A, R* L) {
#pragma unroll
    for (int j = 0; j < N; ++j) {
        R s = A[j * N + j];
#pragma unroll
        for (int k = 0; k < j; ++k) s -= L[j * N + k] * L[j * N + k];
        if (!(s > R(0)) || !is_finite(s)) return false;
        const R ljj = sqrt(s);
        L[j * N + j] = ljj;
        const R inv = R(1) / ljj;
#pragma unroll
        for (int i = j + 1; i < N; ++i) {
            R t = R(0.5) * (A[i * N + j] + A[j * N + i]);
#pragma unroll
            for (int k = 0; k < j; ++k) t -= L[i * N + k] * L[j * N + k];
            L[i * N + j] = t * inv;
        }
#pragma unroll
        for (int i = 0; i < j; ++i) L[i * N + j] = R(0);
    }
    return true;
}

// X[r][:] = A^-1 Bm[r][:] for r < ROWS, with L the Cholesky factor of A (N x N): X = Bm A^-1 for symmetric A
template <int ROWS, int N, class R>
RXGD_HD void solve_rows(const R* L, const R* Bm, R* X) {
#pragma unroll
    for (int r = 0; r < ROWS; ++r) {
        R z[N];
#pragma unroll
        for (int i = 0; i < N; ++i) {
            R s = Bm[r * N + i];
#pragma unroll
            for (int k = 0; k < i; ++k) s -= L[i * N + k] * z[k];
            z[i] = s / L[i * N + i];
        }
#pragma unroll
        for (int i = N - 1; i >= 0; --i) {
            R s = z[i];
#pragma unroll
            for (int k = i + 1; k < N; ++k) s -= L[k * N + i] * X[r * N + k];
            X[r * N + i] = s / L[i * N + i];
        }
    }
}

template <int N, class R>
RXGD_HD void symmetrize(R* S) {
#pragma unroll
    for (int i = 0; i < N; ++i)
#pragma unroll
        for (int j = i + 1; j < N; ++j) {
            const R s = R(0.5) * (S[i * N + j] + S[j * N + i]);
            S[i * N + j] = s; S[j * N + i] = s;
        }
}

// ------------------------------------------------------------------ moment approximation of z = h(x), x ~ N(mu, S)
// Out: mz[K], Szz[K][K], Sxz[N][K].  H::eval<S>(const S* x, S* z) is the user function.

// Linearization (fp32): h(mu), J S J', S J' with the Jacobian J[K][N] from one dual-number evaluation.
template <int N, int K, class H>
RXGD_HD bool moments_lin(const float* mu, const float* S, float* mz, float* Szz, float* Sxz) {
    Dual<N> x[N], z[K];
#pragma unroll
    for (int i = 0; i < N; ++i) { x[i] = Dual<N>(mu[i]); x[i].g[i] = 1.f; }
    H::eval(x, z);
#pragma unroll
    for (int k = 0; k < K; ++k) mz[k] = z[k].v;
#pragma unroll
    for (int i = 0; i < N; ++i)
#pragma unroll
        for (int k = 0; k < K; ++k) {
            float s = 0.f;
#pragma unroll
            for (int j = 0; j < N; ++j) s += S[i * N + j] * z[k].g[j];
            Sxz[i * K + k] = s;
        }
#pragma unroll
    for (int k = 0; k < K; ++k)
#pragma unroll
        for (int l = 0; l < K; ++l) {
            float s = 0.f;
#pragma unroll
            for (int i = 0; i < N; ++i) s += z[k].g[i] * Sxz[i * K + l];
            Szz[k * K + l] = s;
        }
    symmetrize<K>(Szz);
    return true;
}

// Unscented transform (fp64), 2N + 1 sigma points mu, mu +- sqrt(N + lambda) L[:, i] with L L' = S and
// lambda = alpha^2 (N + kappa) - N (Julier & Uhlmann; the weights of Wan & van der Merwe, 2000):
//   Wm_0 = lambda / (N + lambda), Wc_0 = Wm_0 + 1 - alpha^2 + beta, W_i = 1 / (2 (N + lambda)).
// The moments are accumulated as deviations from h(mu), which the weights allow because they sum to one:
// with alpha = 1e-3 the weights are about +-1e6 / N and the weighted sum of h itself would cancel to a
// relative 1e-10 even in fp64.
template <int N, int K, class H>
RXGD_HD bool moments_ut(const double* mu, const double* S, double alpha, double beta, double kappa, double* mz,
                        double* Szz, double* Sxz) {
    const double lam = alpha * alpha * (N + kappa) - N;
    const double c = N + lam;
    double cS[N * N], L[N * N];
#pragma unroll
    for (int i = 0; i < N * N; ++i) cS[i] = c * S[i];
    if (!(c > 0.0) || !cholesky<N>(cS, L)) {      // S not SPD: the outputs are NaN, never uninitialised
        const double nan = 0.0 / 0.0;
#pragma unroll
        for (int k = 0; k < K; ++k) mz[k] = nan;
#pragma unroll
        for (int i = 0; i < K * K; ++i) Szz[i] = nan;
#pragma unroll
        for (int i = 0; i < N * K; ++i) Sxz[i] = nan;
        return false;
    }
    const double wi = 0.5 / c;
    const double wc0 = lam / c + 1.0 - alpha * alpha + beta;
    double z0[K], dp[N][K], dm[N][K];
    H::eval(mu, z0);
#pragma unroll 1         // one sigma pair at a time: unrolling 2N user-function evaluations only grows the code
    for (int i = 0; i < N; ++i) {
        double xp[N], xm[N], zp[K], zm[K];
#pragma unroll
        for (int j = 0; j < N; ++j) { xp[j] = mu[j] + L[j * N + i]; xm[j] = mu[j] - L[j * N + i]; }
        H::eval(xp, zp);
        H::eval(xm, zm);
#pragma unroll
        for (int k = 0; k < K; ++k) { dp[i][k] = zp[k] - z0[k]; dm[i][k] = zm[k] - z0[k]; }
    }
    double e[K];          // mz - h(mu) = W_i sum_i (dp_i + dm_i)
#pragma unroll
    for (int k = 0; k < K; ++k) {
        double s = 0.0;
#pragma unroll
        for (int i = 0; i < N; ++i) s += dp[i][k] + dm[i][k];
        e[k] = wi * s;
        mz[k] = z0[k] + e[k];
    }
    // Szz = Wc_0 (z0 - mz)(z0 - mz)' + W_i sum_i [(zp_i - mz)(zp_i - mz)' + (zm_i - mz)(zm_i - mz)'], z0 - mz = -e
#pragma unroll
    for (int k = 0; k < K; ++k)
#pragma unroll
        for (int l = 0; l <= k; ++l) {
            double s = 0.0;
#pragma unroll
            for (int i = 0; i < N; ++i)
                s += (dp[i][k] - e[k]) * (dp[i][l] - e[l]) + (dm[i][k] - e[k]) * (dm[i][l] - e[l]);
            const double v = wc0 * e[k] * e[l] + wi * s;
            Szz[k * K + l] = v; Szz[l * K + k] = v;
        }
    // Sxz = W_i sum_i L[:, i] (zp_i - zm_i)'   (the centre point has no x deviation)
#pragma unroll
    for (int j = 0; j < N; ++j)
#pragma unroll
        for (int k = 0; k < K; ++k) {
            double s = 0.0;
#pragma unroll
            for (int i = 0; i < N; ++i) s += L[j * N + i] * (dp[i][k] - dm[i][k]);
            Sxz[j * K + k] = wi * s;
        }
    return true;
}

// ------------------------------------------------------------------ the chain steps
// C (the generated configuration) provides: D, M, METHOD, HAS_G, ALPHA, BETA, KAPPA, types F and G.
template <class C> struct Steps {
    typedef typename RealOf<C::METHOD>::T R;
    enum { D = C::D, M = C::M };

    template <int N, int K, class H>
    RXGD_HD static bool moments(const R* mu, const R* S, R* mz, R* Szz, R* Sxz) {
        if constexpr ((int)C::METHOD == (int)UNSCENTED) return moments_ut<N, K, H>(mu, S, C::ALPHA, C::BETA, C::KAPPA, mz, Szz, Sxz);
        else return moments_lin<N, K, H>(mu, S, mz, Szz, Sxz);
    }

    // Prediction through the transition: mp = E[f(x)], Sp = Cov[f(x)] + P, Sxz = Cov[x, f(x)]; Lp = chol(Sp)
    RXGD_HD static int predict(const R* m, const R* S, const float* P, R* mp, R* Sp, R* Sxz, R* Lp) {
        if (!moments<D, D, typename C::F>(m, S, mp, Sp, Sxz)) return ERR_NOT_SPD;
#pragma unroll
        for (int i = 0; i < D * D; ++i) Sp[i] += (R)P[i];
        return cholesky<D>(Sp, Lp) ? OK : ERR_NOT_SPD;
    }

    // Observation update of N(m, S) (in place) by y ~ N(B x, Q) or N(g(x), Q)
    RXGD_HD static int update(R* m, R* S, const float* y, const float* B, const float* Q) {
        R my[M], Syy[M * M], Sxy[D * M];
        if constexpr (C::HAS_G) {
            if (!moments<D, M, typename C::G>(m, S, my, Syy, Sxy)) return ERR_NOT_SPD;
        } else {
#pragma unroll
            for (int k = 0; k < M; ++k) {
                R s = R(0);
#pragma unroll
                for (int j = 0; j < D; ++j) s += (R)B[k * D + j] * m[j];
                my[k] = s;
            }
#pragma unroll
            for (int i = 0; i < D; ++i)
#pragma unroll
                for (int k = 0; k < M; ++k) {
                    R s = R(0);
#pragma unroll
                    for (int j = 0; j < D; ++j) s += S[i * D + j] * (R)B[k * D + j];
                    Sxy[i * M + k] = s;
                }
#pragma unroll
            for (int k = 0; k < M; ++k)
#pragma unroll
                for (int l = 0; l < M; ++l) {
                    R s = R(0);
#pragma unroll
                    for (int j = 0; j < D; ++j) s += (R)B[k * D + j] * Sxy[j * M + l];
                    Syy[k * M + l] = s;
                }
        }
#pragma unroll
        for (int i = 0; i < M * M; ++i) Syy[i] += (R)Q[i];
        return gain_update(m, S, y, my, Syy, Sxy);
    }

    // m += K (y - my), S -= K Syy K' with K = Sxy Syy^-1
    RXGD_HD static int gain_update(R* m, R* S, const float* y, const R* my, const R* Syy, const R* Sxy) {
        R Ly[M * M], K[D * M];
        if (!cholesky<M>(Syy, Ly)) return ERR_NOT_SPD;
        solve_rows<D, M>(Ly, Sxy, K);
#pragma unroll
        for (int i = 0; i < D; ++i) {
            R s = R(0);
#pragma unroll
            for (int k = 0; k < M; ++k) s += K[i * M + k] * ((R)y[k] - my[k]);
            m[i] += s;
        }
#pragma unroll
        for (int i = 0; i < D; ++i)
#pragma unroll
            for (int j = 0; j < D; ++j) {
                R s = R(0);
#pragma unroll
                for (int k = 0; k < M; ++k) s += K[i * M + k] * Sxy[j * M + k];     // K Syy K' = K Sxy'
                S[i * D + j] -= s;
            }
        symmetrize<D>(S);
        return OK;
    }

    // RTS backward step from the filtered (mf, Sf) of step t and the smoothed (ms, Ss) of step t + 1 (in place):
    // G = Sxz Sp^-1, ms <- mf + G (ms - mp), Ss <- Sf + G (Ss - Sp) G'
    RXGD_HD static int smooth_back(const R* mf, const R* Sf, const float* P, R* ms, R* Ss) {
        R mp[D], Sp[D * D], Sxz[D * D], Lp[D * D], G[D * D];
        const int rc = predict(mf, Sf, P, mp, Sp, Sxz, Lp);
        if (rc != OK) return rc;
        solve_rows<D, D>(Lp, Sxz, G);
        R dm[D], W[D * D];
#pragma unroll
        for (int i = 0; i < D; ++i) dm[i] = ms[i] - mp[i];
#pragma unroll
        for (int i = 0; i < D; ++i) {
            R s = R(0);
#pragma unroll
            for (int j = 0; j < D; ++j) s += G[i * D + j] * dm[j];
            ms[i] = mf[i] + s;
        }
#pragma unroll
        for (int i = 0; i < D; ++i)           // W = (Ss - Sp) G'
#pragma unroll
            for (int j = 0; j < D; ++j) {
                R s = R(0);
#pragma unroll
                for (int k = 0; k < D; ++k) s += (Ss[i * D + k] - Sp[i * D + k]) * G[j * D + k];
                W[i * D + j] = s;
            }
#pragma unroll
        for (int i = 0; i < D; ++i)
#pragma unroll
            for (int j = 0; j < D; ++j) {
                R s = R(0);
#pragma unroll
                for (int k = 0; k < D; ++k) s += G[i * D + k] * W[k * D + j];
                Ss[i * D + j] = Sf[i * D + j] + s;
            }
        symmetrize<D>(Ss);
        return OK;
    }

    // One datum of the Delta transition observed as y ~ N(c' x, 1/tau), tau ~ Gamma(shape, rate), constraint
    // q(x, tau) = q(x) q(tau) (M = 1, c = B).  In: (m, S) = the prediction N(E f(x_prev), Cov f(x_prev) + P), the
    // message through the Delta node, fixed within the datum; (a, b) = the Gamma prior, which is also the initial
    // q(tau).  Out: q(x) = (m, S) and q(tau) = (a, b) after `iters` VMP iterations, each of which updates
    //   q(x) ∝ N(x | m, S) N(y | c' x, 1 / E[tau]),   then   q(tau) = Gamma(a0 + 1/2, b0 + E_q[(y - c' x)^2] / 2).
    RXGD_HD static int vmp_gamma(R* m, R* S, float y, const float* c, R& a, R& b, int iters) {
        const R a0 = a, b0 = b;
        R mp[D], Sp[D * D], Sc[D];
#pragma unroll
        for (int i = 0; i < D; ++i) mp[i] = m[i];
#pragma unroll
        for (int i = 0; i < D * D; ++i) Sp[i] = S[i];
#pragma unroll
        for (int i = 0; i < D; ++i) {
            R s = R(0);
#pragma unroll
            for (int j = 0; j < D; ++j) s += Sp[i * D + j] * (R)c[j];
            Sc[i] = s;
        }
        R cSc = R(0), cm = R(0);
#pragma unroll
        for (int i = 0; i < D; ++i) { cSc += (R)c[i] * Sc[i]; cm += (R)c[i] * mp[i]; }
        for (int it = 0; it < iters; ++it) {
            const R s = cSc + b / a;                 // innovation variance c' Sp c + 1 / E[tau]
            if (!(s > R(0))) return ERR_NOT_SPD;
            const R r = ((R)y - cm) / s;
#pragma unroll
            for (int i = 0; i < D; ++i) m[i] = mp[i] + Sc[i] * r;
#pragma unroll
            for (int i = 0; i < D; ++i)
#pragma unroll
                for (int j = 0; j < D; ++j) S[i * D + j] = Sp[i * D + j] - Sc[i] * Sc[j] / s;
            R cmq = R(0), cSqc = R(0);
#pragma unroll
            for (int i = 0; i < D; ++i) {
                cmq += (R)c[i] * m[i];
                R t = R(0);
#pragma unroll
                for (int j = 0; j < D; ++j) t += S[i * D + j] * (R)c[j];
                cSqc += (R)c[i] * t;
            }
            const R e = (R)y - cmq;
            a = a0 + R(0.5);
            b = b0 + R(0.5) * (e * e + cSqc);
        }
        return OK;
    }
};

// ------------------------------------------------------------------ kernels (one thread per chain, SoA [..][batch])
// Model constants shared by every chain, passed by value: row-major m0[D], S0[D][D], P[D][D], B[M][D], Q[M][M].
struct Params {
    float m0[8], S0[64], P[64], B[64], Q[64];
};

template <int N, class R> RXGD_HD void load_gauss(const float* mean, const float* cov, long long t, long long batch,
                                                  long long b, R* m, R* S) {
#pragma unroll
    for (int i = 0; i < N; ++i) m[i] = (R)mean[(t * N + i) * batch + b];
#pragma unroll
    for (int i = 0; i < N * N; ++i) S[i] = (R)cov[(t * N * N + i) * batch + b];
}
template <int N, class R> RXGD_HD int store_gauss(float* mean, float* cov, long long t, long long batch, long long b,
                                                  const R* m, const R* S) {
    bool fin = true;
#pragma unroll
    for (int i = 0; i < N; ++i) { mean[(t * N + i) * batch + b] = (float)m[i]; fin = fin && is_finite(m[i]); }
#pragma unroll
    for (int i = 0; i < N * N; ++i) { cov[(t * N * N + i) * batch + b] = (float)S[i]; fin = fin && is_finite(S[i]); }
    return fin ? OK : ERR_NAN;
}
// the fp32 value a stored carry takes: rounding every step makes a chunked run equal a single call
template <int N, class R> RXGD_HD void round_f32(R* a) {
#pragma unroll
    for (int i = 0; i < N; ++i) a[i] = (R)(float)a[i];
}

// Whole series: EKF / UKF forward (prior on x[1], observation at every step, x[t] = f(x[t-1]) + N(0, P)), the
// filtered marginals written to post (and filt), then ERTS / URTS backward over them.
template <class C>
RXGD_HD void smooth_chain(const Params& p, int T, long long batch, long long b, const float* y, const unsigned char* ymask,
                          float* post_mean, float* post_cov, float* filt_mean, float* filt_cov, int* status) {
    typedef Steps<C> St;
    typedef typename St::R R;
    enum { D = C::D, M = C::M };
    int st = OK;
    R m[D], S[D * D];
#pragma unroll
    for (int i = 0; i < D; ++i) m[i] = (R)p.m0[i];
#pragma unroll
    for (int i = 0; i < D * D; ++i) S[i] = (R)p.S0[i];
    for (int t = 0; t < T; ++t) {
        if (t > 0) {
            R mp[D], Sxz[D * D], Lp[D * D];
            R Sp[D * D];
            const int rc = St::predict(m, S, p.P, mp, Sp, Sxz, Lp);
            if (rc != OK && st == OK) st = rc;
#pragma unroll
            for (int i = 0; i < D; ++i) m[i] = mp[i];
#pragma unroll
            for (int i = 0; i < D * D; ++i) S[i] = Sp[i];
        }
        if (!ymask || ymask[(long long)t * batch + b]) {
            float yt[M];
#pragma unroll
            for (int k = 0; k < M; ++k) yt[k] = y[((long long)t * M + k) * batch + b];
            const int rc = St::update(m, S, yt, p.B, p.Q);
            if (rc != OK && st == OK) st = rc;
        }
        int rc = store_gauss<D>(post_mean, post_cov, t, batch, b, m, S);
        if (filt_mean) store_gauss<D>(filt_mean, filt_cov, t, batch, b, m, S);
        if (rc != OK && st == OK) st = rc;
    }
    for (int t = T - 2; t >= 0; --t) {        // m, S: the smoothed marginal of step t + 1
        R mf[D], Sf[D * D];
        load_gauss<D>(post_mean, post_cov, t, batch, b, mf, Sf);
        int rc = St::smooth_back(mf, Sf, p.P, m, S);
        if (rc != OK && st == OK) st = rc;
        rc = store_gauss<D>(post_mean, post_cov, t, batch, b, m, S);
        if (rc != OK && st == OK) st = rc;
    }
    if (status) status[b] = st;
}

// One time-chunk of the streaming filter.  Carry q(x) = carry_mean[D][batch], carry_cov[D][D][batch] (in / out) and,
// with carry_tau != null (M = 1), q(tau) = (shape, rate) as carry_tau[2][batch] with `iters` VMP iterations per datum;
// otherwise the observation noise is Q.  Every datum first pushes the carry through the transition.
template <class C>
RXGD_HD void filter_chain(const Params& p, int T, long long batch, long long b, const float* y, const unsigned char* ymask,
                          float* carry_mean, float* carry_cov, float* carry_tau, int iters, float* filt_mean,
                          float* filt_cov, float* filt_tau, int* status) {
    typedef Steps<C> St;
    typedef typename St::R R;
    enum { D = C::D, M = C::M };
    int st = OK;
    R m[D], S[D * D], ab[2] = {R(0), R(0)};
    load_gauss<D>(carry_mean, carry_cov, 0, batch, b, m, S);
    if (carry_tau) { ab[0] = (R)carry_tau[b]; ab[1] = (R)carry_tau[batch + b]; }
    for (int t = 0; t < T; ++t) {
        R mp[D], Sp[D * D], Sxz[D * D], Lp[D * D];
        int rc = St::predict(m, S, p.P, mp, Sp, Sxz, Lp);
        if (rc != OK && st == OK) st = rc;
#pragma unroll
        for (int i = 0; i < D; ++i) m[i] = mp[i];
#pragma unroll
        for (int i = 0; i < D * D; ++i) S[i] = Sp[i];
        if (!ymask || ymask[(long long)t * batch + b]) {
            float yt[M];
#pragma unroll
            for (int k = 0; k < M; ++k) yt[k] = y[((long long)t * M + k) * batch + b];
            if constexpr (M == 1 && !C::HAS_G) {
                if (carry_tau) rc = St::vmp_gamma(m, S, yt[0], p.B, ab[0], ab[1], iters);
                else rc = St::update(m, S, yt, p.B, p.Q);
            } else {
                rc = St::update(m, S, yt, p.B, p.Q);
            }
            if (rc != OK && st == OK) st = rc;
        }
        round_f32<D>(m);
        round_f32<D * D>(S);
        round_f32<2>(ab);
        if (filt_mean) {
            rc = store_gauss<D>(filt_mean, filt_cov, t, batch, b, m, S);
            if (rc != OK && st == OK) st = rc;
        }
        if (filt_tau) { filt_tau[(2LL * t) * batch + b] = (float)ab[0]; filt_tau[(2LL * t + 1) * batch + b] = (float)ab[1]; }
    }
    const int rc = store_gauss<D>(carry_mean, carry_cov, 0, batch, b, m, S);
    if (rc != OK && st == OK) st = rc;
    if (carry_tau) {
        carry_tau[b] = (float)ab[0]; carry_tau[batch + b] = (float)ab[1];
        if ((!is_finite(ab[0]) || !is_finite(ab[1])) && st == OK) st = ERR_NAN;
    }
    if (status) status[b] = st;
}

}  // namespace rxgd
