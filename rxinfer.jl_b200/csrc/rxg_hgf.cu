// Variational (VMP) members of the hot path: the GCV node of the Hierarchical Gaussian Filter
// (SURVEY.md section 8a row 10) and the Gamma-precision rules around a scalar smoother (row 9).
//
// HGF: per datum the reference's streaming engine [ref: /root/reference/src/inference/
// streaming.jl:349-407] runs `iterations` VMP sweeps over the 5-node graph of
// test/models/statespace/hgf_tests.jl:10-31 with q(xt, xt_min) q(zt) and GCVMetadata(
// GaussHermiteCubature(31)) (hgf_tests.jl:33-40), then @autoupdates carry q(zt), q(xt) into the
// next step's priors (hgf_tests.jl:46-49).  hgf_filter_kernel fuses T steps x iters sweeps per
// chain into one launch; state lives in registers, the 31 exp(-kappa z_i) factors that do not
// change across the iterations of a step are hoisted.  This family is SFU/FP32-issue bound
// (~21 + 31*iters exp per step against 20 bytes of I/O), not HBM bound.
#include <math.h>

#include "rxg_internal.h"

namespace rxg {

__constant__ float c_gh_t[31];    // Gauss-Hermite nodes (physicists')
__constant__ float c_gh_lw[31];   // log weights
__constant__ float c_gh_lw2[31];  // log2 weights (for the ex2-based inner loop)

// Gauss-Hermite nodes/weights by Newton iteration on the orthonormal recurrence (host, fp64): the textbook scheme
// (Press et al., Numerical Recipes, `gauher`; the starting guesses 1.85575 / 1.14 / 0.426 / 1.86 / 1.91 are that routine's).
// Third-party algorithm, not from the reference -- ReactiveMP's GaussHermiteCubature takes its nodes from FastGaussQuadrature.
void gauss_hermite_31(double* t, double* w) {
    const int n = 31;
    const double pim4 = 0.7511255444649425;
    double z = 0, z1, pp = 0;
    const int m = (n + 1) / 2;
    for (int i = 0; i < m; ++i) {
        if (i == 0) z = sqrt(2.0 * n + 1.0) - 1.85575 * pow(2.0 * n + 1.0, -0.16667);
        else if (i == 1) z -= 1.14 * pow((double)n, 0.426) / z;
        else if (i == 2) z = 1.86 * z - 0.86 * t[0];
        else if (i == 3) z = 1.91 * z - 0.91 * t[1];
        else z = 2.0 * z - t[i - 2];
        for (int its = 0; its < 200; ++its) {
            double p1 = pim4, p2 = 0.0;
            for (int j = 0; j < n; ++j) {
                double p3 = p2; p2 = p1;
                p1 = z * sqrt(2.0 / (j + 1)) * p2 - sqrt((double)j / (j + 1)) * p3;
            }
            pp = sqrt(2.0 * n) * p2;
            z1 = z; z = z1 - p1 / pp;
            if (fabs(z - z1) <= 1e-15 * fabs(z) + 1e-300) break;
        }
        t[i] = z; t[n - 1 - i] = -z;
        w[i] = 2.0 / (pp * pp); w[n - 1 - i] = w[i];
    }
}

int ensure_gh_tables(rxg_ctx* ctx) {
    if (ctx->gh_ready) return RXG_OK;
    double t[31], w[31];
    gauss_hermite_31(t, w);
    float tf[31], lw[31], lw2[31];
    for (int i = 0; i < 31; ++i) { tf[i] = (float)t[i]; lw[i] = (float)log(w[i]); lw2[i] = (float)log2(w[i]); }
    RXG_CUDA(ctx, cudaMemcpyToSymbol(c_gh_t, tf, sizeof(tf)));
    RXG_CUDA(ctx, cudaMemcpyToSymbol(c_gh_lw, lw, sizeof(lw)));
    RXG_CUDA(ctx, cudaMemcpyToSymbol(c_gh_lw2, lw2, sizeof(lw2)));
    ctx->gh_ready = true;
    return RXG_OK;
}

struct GcvJoint { float m1, m2, V11, V12, V22; };

// @marginalrule GCV(:y_x): W = [[w_y + g, -g], [-g, w_x + g]], xi = [xi_y, xi_x].
// det = w_y w_x + g (w_y + w_x) is formed without the cancellation of (w_y + g)(w_x + g) - g^2 (g can exceed
// w_y, w_x by orders of magnitude when the volatility level is low).
__device__ __forceinline__ GcvJoint gcv_joint(float xiy, float wy, float xix, float wx, float g) {
    const float a = wy + g, c = wx + g;
    const float det = __fmaf_rn(g, wy + wx, wy * wx);
    const float r = 1.0f / det;
    GcvJoint j;
    j.V11 = c * r; j.V12 = g * r; j.V22 = a * r;
    j.m1 = __fmaf_rn(j.V11, xiy, j.V12 * xix);
    j.m2 = __fmaf_rn(j.V12, xiy, j.V22 * xix);
    return j;
}
// psi = E[(y - x)^2] under the joint = (m1 - m2)^2 + V11 + V22 - 2 V12, in closed form: the variance part is
// (w_y + w_x) / det and the mean difference w_y w_x (m_y - m_x) / det -- no subtraction of nearly equal numbers.
__device__ __forceinline__ float gcv_psi(float my, float wy, float mx, float wx, float g) {
    const float r = 1.0f / __fmaf_rn(g, wy + wx, wy * wx);
    const float dm = wy * wx * (my - mx) * r;
    return __fmaf_rn(dm, dm, (wy + wx) * r);
}
// A * B of the node with PointMass kappa, omega
__device__ __forceinline__ float gcv_gamma(float mz, float vz, float kappa, float omega) {
    return expf(-omega - kappa * mz + 0.5f * kappa * kappa * vz);
}

// prod(Normal(mu0, v0), ELQ(a = kappa, b, c = -kappa, d = 0)) by GH-31 moment matching.
// ez[i] = exp(-kappa z_i) precomputed; shift = expansion point for the second moment.
__device__ __forceinline__ void gh_moment_match(const float* ez, float mu0, float s, float kappa, float b,
                                                float shift, float& mz, float& vz) {
    float lmax = -INFINITY;
#pragma unroll
    for (int i = 0; i < 31; ++i) {
        const float z = __fmaf_rn(s, c_gh_t[i], mu0);
        const float l = c_gh_lw[i] - 0.5f * __fmaf_rn(b, ez[i], kappa * z);
        lmax = fmaxf(lmax, l);
    }
    float S0 = 0.f, S1 = 0.f, S2 = 0.f;
#pragma unroll
    for (int i = 0; i < 31; ++i) {
        const float z = __fmaf_rn(s, c_gh_t[i], mu0);
        const float l = c_gh_lw[i] - 0.5f * __fmaf_rn(b, ez[i], kappa * z);
        const float e = __expf(l - lmax);
        const float u = z - shift;
        S0 += e;
        S1 = __fmaf_rn(e, u, S1);
        S2 = __fmaf_rn(e * u, u, S2);
    }
    const float r = 1.0f / S0;
    const float du = S1 * r;
    mz = shift + du;
    vz = __fmaf_rn(-du, du, S2 * r);
}

__device__ __forceinline__ float ex2_approx(float x) {
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}

// Fused HGF filter.  Per step the Gaussian factor of the z-product (prior pushed through the random
// walk) is fixed across the VMP iterations, so everything that depends only on the 31 quadrature
// nodes is hoisted out of the iteration loop: z_i - mu0, exp(-kappa z_i) and the log2-domain
// constant c2_i = log2 w_i - (kappa log2e / 2) z_i.  One iteration then costs, per node,
//   pass 1:  l_i = fma(b2, ez_i, c2_i); lmax = max(lmax, l_i)                       (2 instr)
//   pass 2:  e = ex2(l_i - lmax); w = u_i - delta; S0 += e; S1 += e w; S2 += e w w  (8 instr, 1 MUFU)
// with b2 = -(log2e / 2) psi A and delta = previous iterate minus prior mean (moments are
// accumulated around the previous iterate, which removes the fp32 cancellation in the variance).
//
// FE: Bethe free energy of each datum's graph after every VMP iteration, fe[T][iters][batch]
// [ref: definition /root/reference/src/model/plugins/reactivemp_free_energy.jl:84-126; the reference pins its average
//  over the data for this model, test/models/statespace/hgf_tests.jl:112-119].  Single-variable clusters cancel, leaving
//   F = U[zt_min prior] + U[xt_min prior] + U[zt | zt_min] + U[GCV] + U[y | xt] - H[q(zt, zt_min)] - H[q(xt, xt_min)],
// where q(zt, zt_min) is the (out, mu) marginal of the Normal node whose inbound message on `out` is the GCV node's
// ExponentialLinearQuadratic read through mean_var: GaussHermiteCubature(31) against N(0, 1) with the density
// re-weighted by exp(z^2 / 2) -- nodes sqrt(2) t_i are fixed, so exp(-kappa z_i) and the log-weights are per-launch
// constants kept in shared memory (s_e0, s_c0).  All differences of nearly equal terms are taken in closed form.
template <bool FE>
__global__ void __launch_bounds__(64)
hgf_filter_kernel(const float* __restrict__ y, float* __restrict__ out, int T, int64_t batch, int iters,
                  float kappa, float omega, float zvar, float yvar, float i_mz, float i_vz, float i_mx,
                  float i_vx, const float* __restrict__ prev, float* __restrict__ fe) {
    __shared__ float s_e0[32], s_c0[32], s_z0[32];
    if (FE) {
        if (threadIdx.x < 31) {
            const float z = 1.41421356237309505f * c_gh_t[threadIdx.x];
            s_z0[threadIdx.x] = z;
            s_e0[threadIdx.x] = expf(-kappa * z);
            s_c0[threadIdx.x] = c_gh_lw[threadIdx.x] + 0.5f * z * z - 0.5f * kappa * z;     // log w_i + z^2/2 - kappa z / 2
        }
        __syncthreads();
    }
    const int64_t b = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= batch) return;
    constexpr float LOG2E = 1.4426950408889634f;
    constexpr float LOG_2PI = 1.8378770664093453f;
    if (prev) {   // streaming carry: out[T-1] of the previous chunk, rows (m_x, v_x, m_z, v_z)
        i_mx = __ldg(prev + b); i_vx = __ldg(prev + batch + b);
        i_mz = __ldg(prev + 2 * batch + b); i_vz = __ldg(prev + 3 * batch + b);
    }
    float mzp = i_mz, vzp = i_vz, mxp = i_mx, vxp = i_vx;
    float mz = i_mz, vz = i_vz;                 // q(zt), carried across iterations and steps
    const float wy = 1.0f / yvar;
    const float eA = expf(-omega);
    const float hk2 = 0.5f * LOG2E * kappa;
    float ynext = __ldg(y + b);
    for (int t = 0; t < T; ++t) {
        const float yt = ynext;
        if (t + 1 < T) ynext = __ldg(y + (int64_t)(t + 1) * batch + b);
        // zt ~ Normal(zt_min, z_variance): message into zt from the prior side
        const float mu0 = mzp, v0 = vzp + zvar;
        const float s = sqrtf(2.0f * v0);
        float ez[31], c2[31], u[31];
#pragma unroll
        for (int i = 0; i < 31; ++i) {
            u[i] = s * c_gh_t[i];
            const float z = mu0 + u[i];
            ez[i] = expf(-kappa * z);
            c2[i] = __fmaf_rn(-hk2, z, c_gh_lw2[i]);
        }
        const float wx = 1.0f / vxp;
        const float xiy = yt * wy, xix = mxp * wx;
        GcvJoint j;
        for (int it = 0; it < iters; ++it) {
            const float g = gcv_gamma(mz, vz, kappa, omega);
            j = gcv_joint(xiy, wy, xix, wx, g);
            const float psi = gcv_psi(yt, wy, mxp, wx, g);
            const float b2 = -0.5f * LOG2E * psi * eA;
            float lmax = -INFINITY;
#pragma unroll
            for (int i = 0; i < 31; ++i) lmax = fmaxf(lmax, __fmaf_rn(b2, ez[i], c2[i]));
            const float delta = mz - mu0;
            float S0 = 0.f, S1 = 0.f, S2 = 0.f;
#pragma unroll
            for (int i = 0; i < 31; ++i) {
                const float e = ex2_approx(__fmaf_rn(b2, ez[i], c2[i]) - lmax);
                const float w = u[i] - delta;
                S0 += e;
                S1 = __fmaf_rn(e, w, S1);
                S2 = __fmaf_rn(e * w, w, S2);
            }
            const float r = 1.0f / S0;
            const float dw = S1 * r;
            mz = mz + dw;
            vz = __fmaf_rn(-dw, dw, S2 * r);
            if (FE) {
                // mean_var(ELQ(kappa, psi A, -kappa, 0)) by GH-31 against N(0, 1), pdf re-weighted by exp(z^2 / 2)
                const float hb = -0.5f * psi * eA;
                float lm = -INFINITY;
#pragma unroll
                for (int i = 0; i < 31; ++i) lm = fmaxf(lm, __fmaf_rn(hb, s_e0[i], s_c0[i]));
                float T0 = 0.f, T1 = 0.f, T2 = 0.f;
#pragma unroll
                for (int i = 0; i < 31; ++i) {
                    const float e = __expf(__fmaf_rn(hb, s_e0[i], s_c0[i]) - lm);
                    const float z = s_z0[i];
                    T0 += e; T1 = __fmaf_rn(e, z, T1); T2 = __fmaf_rn(e * z, z, T2);
                }
                const float me = T1 / T0;
                const float ve = fmaxf(__fmaf_rn(-me, me, T2 / T0), 1e-30f);
                // q(zt, zt_min) = N(zt_min; mzp, vzp) N(zt; zt_min, zvar) N(zt; me, ve)
                const float iz = 1.0f / zvar, ie = 1.0f / ve, ip = 1.0f / vzp;
                const float w11 = iz + ie, w22 = ip + iz;
                const float detz = __fmaf_rn(iz, ip + ie, ie * ip);             // w11 w22 - iz^2, cancellation free
                const float rz = 1.0f / detz;
                const float v22 = w11 * rz;
                const float xi1 = me * ie, xi2 = mzp * ip;
                const float j2 = (iz * xi1 + w11 * xi2) * rz;
                const float dj = (ip * xi1 - ie * xi2) * rz;                     // E zt - E zt_min
                const float U_nz = 0.5f * (LOG_2PI + logf(zvar)) + 0.5f * __fmaf_rn(dj, dj, (ip + ie) * rz) * iz;
                const float dz2 = j2 - mzp;
                const float U_pz = 0.5f * (LOG_2PI + logf(vzp)) + 0.5f * __fmaf_rn(dz2, dz2, v22) * ip;
                const float dx2 = j.m2 - mxp;
                const float U_px = 0.5f * (LOG_2PI + logf(vxp)) + 0.5f * __fmaf_rn(dx2, dx2, j.V22) * wx;
                const float Bn = expf(-kappa * mz + 0.5f * kappa * kappa * vz);
                const float U_g = 0.5f * (LOG_2PI + (kappa * mz + omega) + psi * eA * Bn);
                const float dy = yt - j.m1;
                const float U_o = 0.5f * (LOG_2PI + logf(yvar)) + 0.5f * __fmaf_rn(dy, dy, j.V11) * wy;
                const float detx = __fmaf_rn(g, wy + wx, wy * wx);
                const float H_z = LOG_2PI + 1.0f - 0.5f * logf(detz);           // 1/2 log((2 pi e)^2 / det W)
                const float H_x = LOG_2PI + 1.0f - 0.5f * logf(detx);
                fe[((int64_t)t * iters + it) * batch + b] = U_nz + U_pz + U_px + U_g + U_o - H_z - H_x;
            }
        }
        out[((int64_t)t * 4 + 0) * batch + b] = j.m1;
        out[((int64_t)t * 4 + 1) * batch + b] = j.V11;
        out[((int64_t)t * 4 + 2) * batch + b] = mz;
        out[((int64_t)t * 4 + 3) * batch + b] = vz;
        mxp = j.m1; vxp = j.V11; mzp = mz; vzp = vz;
    }
}

// ---- per-rule GCV kernels
__global__ void k_gcv_out(int64_t n, const float* m_x, const float* v_x, const float* m_z, const float* v_z,
                          float kappa, float omega, float* m_out, float* v_out) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    m_out[i] = m_x[i];
    v_out[i] = v_x[i] + 1.0f / gcv_gamma(m_z[i], v_z[i], kappa, omega);
}
__global__ void k_gcv_yx(int64_t n, const float* m_y, const float* v_y, const float* m_x, const float* v_x,
                         const float* m_z, const float* v_z, float kappa, float omega, float* m, float* V) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float wy = 1.0f / v_y[i], wx = 1.0f / v_x[i];
    GcvJoint j = gcv_joint(m_y[i] * wy, wy, m_x[i] * wx, wx, gcv_gamma(m_z[i], v_z[i], kappa, omega));
    m[i] = j.m1; m[n + i] = j.m2;
    V[i] = j.V11; V[n + i] = j.V12; V[2 * n + i] = j.V12; V[3 * n + i] = j.V22;
}
__global__ void k_gcv_z_prod(int64_t n, const float* m_yx, const float* V_yx, const float* m_zp, const float* v_zp,
                             float kappa, float omega, float* m_z, float* v_z) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float dm = m_yx[i] - m_yx[n + i];
    const float psi = __fmaf_rn(dm, dm, V_yx[i] + V_yx[3 * n + i] - V_yx[n + i] - V_yx[2 * n + i]);
    const float mu0 = m_zp[i], v0 = v_zp[i];
    const float s = sqrtf(2.0f * v0);
    float ez[31];
#pragma unroll
    for (int q = 0; q < 31; ++q) ez[q] = expf(-kappa * __fmaf_rn(s, c_gh_t[q], mu0));
    float mz, vz;
    gh_moment_match(ez, mu0, s, kappa, psi * expf(-omega), mu0, mz, vz);
    m_z[i] = mz; v_z[i] = vz;
}

__device__ __forceinline__ float digamma_f(float x) {      // psi(x), x > 0: recurrence up to x >= 6, then the asymptotic series
    float r = 0.f;
    while (x < 6.f) { r -= 1.f / x; x += 1.f; }
    const float i = 1.f / x, i2 = i * i;
    return r + logf(x) - 0.5f * i - i2 * (1.f / 12.f - i2 * (1.f / 120.f - i2 * (1.f / 252.f)));
}
// ---- Gamma-precision VMP around a scalar smoother (d = m = 1), tau shared over time per chain.
// fe[iterations][batch] (optional): Bethe free energy after every iteration, with q(x) the exact chain posterior under the
// E[tau] the sweep ran with and q(tau) the update that followed.  The Gaussian part collapses to the filter's evidence:
//   F = NLE(tau_old) + T/2 (log tau_old - E log tau) + (E tau - tau_old)(b - b0) + KL(q(tau) || Gamma(a0, b0))
// (E_q[-log p(x)] - H[q(x)] = -log Z(tau_old) - sum_t E_q[-log N(y_t; x_t, 1/tau_old)], sum_t E(y_t - x_t)^2 = 2 (b - b0);
// checked against the dense evaluation of the definition in tests/test_oracle_goldens.py)
__global__ void __launch_bounds__(128)
vmp_gamma_kernel(const float* __restrict__ y, float* __restrict__ pm, float* __restrict__ pv,
                 float* __restrict__ shape, float* __restrict__ rate, int T, int64_t batch, int iterations,
                 float a, float vproc, float m0, float v0, float a0, float b0, float init_Etau, float* __restrict__ fe) {
    const int64_t b = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= batch) return;
    float Etau = init_Etau, sh = a0, rt = b0;
    for (int it = 0; it < iterations; ++it) {
        const float q = 1.0f / Etau;       // NormalMeanPrecision(:out)(m_mu, q_tau): variance 1 / E[tau]
        double nle = 0.0;
        float m = m0, v = v0;
        float ynext = __ldg(y + b);
        for (int t = 0; t < T; ++t) {
            const float yt = ynext;
            if (t + 1 < T) ynext = __ldg(y + (int64_t)(t + 1) * batch + b);
            if (t > 0) { m = a * m; v = __fmaf_rn(a * a, v, vproc); }
            const float sinn = v + q;
            const float k = v / sinn;
            if (fe) { const float e = yt - m; nle += 0.5 * (double)(1.8378770664093453f + logf(sinn) + e * e / sinn); }
            m = __fmaf_rn(k, yt - m, m);
            v = __fmaf_rn(-k, v, v);
            pm[(int64_t)t * batch + b] = m;
            pv[(int64_t)t * batch + b] = v;
        }
        float ms = m, vs = v;
        double res;
        { const float d = __ldg(y + (int64_t)(T - 1) * batch + b) - ms; res = (double)__fmaf_rn(d, d, vs); }
        for (int t = T - 2; t >= 0; --t) {
            const float mf = pm[(int64_t)t * batch + b], vf = pv[(int64_t)t * batch + b];
            const float vp = __fmaf_rn(a * a, vf, vproc);
            const float G = a * vf / vp;
            ms = __fmaf_rn(G, ms - a * mf, mf);
            vs = __fmaf_rn(G * G, vs - vp, vf);
            pm[(int64_t)t * batch + b] = ms;
            pv[(int64_t)t * batch + b] = vs;
            const float d = __ldg(y + (int64_t)t * batch + b) - ms;
            res += (double)__fmaf_rn(d, d, vs);
        }
        // prod(Gamma(a0, b0), prod_t NormalMeanPrecision(:tau)(q_out = PointMass y_t, q_mu = q(x_t)))
        const float tau_old = Etau;
        sh = a0 + 0.5f * (float)T;
        rt = b0 + 0.5f * (float)res;
        Etau = sh / rt;
        if (fe) {
            const float Elog = digamma_f(sh) - logf(rt);
            const float kl = (sh - a0) * digamma_f(sh) - lgammaf(sh) + lgammaf(a0) + a0 * (logf(rt) - logf(b0)) + sh * (b0 - rt) / rt;
            fe[(int64_t)it * batch + b] = (float)(nle + 0.5 * T * (double)(logf(tau_old) - Elog) + (double)(Etau - tau_old) * (0.5 * res) + (double)kl);
        }
    }
    shape[b] = sh; rate[b] = rt;
}

// ---- streaming mean-field VMP with a Gamma observation precision (the reference's `test_model1`,
// /root/reference/test/inference/inference_tests.jl:752-775): per datum, `iters` sweeps of
//   q(x_t_min) = N(m_p, v_p) x NormalMeanPrecision(:mu)(q_out = q(x_t))            (prior x backward VMP message)
//   q(x_t)     = NormalMeanPrecision(:out)(q_mu = q(x_t_min)) x NormalMeanPrecision(:mu)(y, q_tau)
//   q(tau)     = Gamma(a_p, b_p) x NormalMeanPrecision(:tau)(q_out = y, q_mu = q(x_t))
// with the priors (m_p, v_p, a_p, b_p) autoupdated from the previous datum's q(x_t), q(tau).
__global__ void __launch_bounds__(128)
stream_vmp_gamma_kernel(const float* __restrict__ y, const float* __restrict__ prev, float* __restrict__ out,
                        float* __restrict__ fe, int T, int64_t batch, int iters, float w, float i_mx, float i_vx,
                        float i_a, float i_b) {
    const int64_t b = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= batch) return;
    float mx = i_mx, vx = i_vx, a = i_a, rt = i_b;
    if (prev) { mx = __ldg(prev + b); vx = __ldg(prev + batch + b); a = __ldg(prev + 2 * batch + b); rt = __ldg(prev + 3 * batch + b); }
    const float iw = 1.0f / w;
    constexpr float LOG_2PI = 1.8378770664093453f;
    float ynext = __ldg(y + b);
    for (int t = 0; t < T; ++t) {
        const float yt = ynext;
        if (t + 1 < T) ynext = __ldg(y + (int64_t)(t + 1) * batch + b);
        const float mp = mx, vp = vx, ap = a, bp = rt;                  // @autoupdates: this datum's priors
        for (int it = 0; it < iters; ++it) {
            // q(x_t_min): precision-weighted product of N(mp, vp) and N(E x_t, 1/w)
            const float wmin = 1.0f / vp + w;
            const float vmin = 1.0f / wmin;
            const float mmin = vmin * __fmaf_rn(mx, w, mp / vp);
            // q(x_t): N(E x_t_min, 1/w) x N(y, 1/E tau)
            const float Etau = a / rt;
            const float wx = w + Etau;
            vx = 1.0f / wx;
            mx = vx * __fmaf_rn(yt, Etau, mmin * w);
            // q(tau): Gamma(ap + 3/2 - 1, bp + ((y - m_x)^2 + v_x) / 2)
            const float d = yt - mx;
            a = ap + 0.5f;
            rt = __fmaf_rn(0.5f, __fmaf_rn(d, d, vx), bp);
            if (fe) {
                const float Et = a / rt, Elog = digamma_f(a) - logf(rt);
                const float dm = mmin - mp, dx = mx - mmin;
                const float U1 = 0.5f * (LOG_2PI + logf(vp)) + __fmaf_rn(dm, dm, vmin) / (2.0f * vp);
                const float U2 = -ap * logf(bp) + lgammaf(ap) - (ap - 1.0f) * Elog + bp * Et;
                const float U3 = 0.5f * (LOG_2PI - logf(w)) + 0.5f * w * (__fmaf_rn(dx, dx, vx) + vmin);
                const float U4 = 0.5f * (LOG_2PI - Elog) + 0.5f * Et * __fmaf_rn(d, d, vx);
                const float Hn = 0.5f * (LOG_2PI + 1.0f + logf(vmin)) + 0.5f * (LOG_2PI + 1.0f + logf(vx));
                const float Hg = a - logf(rt) + lgammaf(a) + (1.0f - a) * digamma_f(a);
                fe[((int64_t)t * iters + it) * batch + b] = U1 + U2 + U3 + U4 - Hn - Hg;
            }
        }
        out[((int64_t)t * 4 + 0) * batch + b] = mx;
        out[((int64_t)t * 4 + 1) * batch + b] = vx;
        out[((int64_t)t * 4 + 2) * batch + b] = a;
        out[((int64_t)t * 4 + 3) * batch + b] = rt;
    }
}

}  // namespace rxg

using namespace rxg;

extern "C" {

int rxg_hgf_filter_fe_f32(rxg_ctx* ctx, int T, int64_t batch, int iters, float kappa, float omega, float z_variance,
                          float y_variance, const float init[4], const float* prev, const float* y, float* out,
                          float* free_energy, unsigned flags) {
    if (!ctx) return RXG_ERR_BAD_ARG;
    if (T < 1 || batch < 1 || iters < 1 || !y || !out || (!init && !prev) || !(z_variance > 0.f) || !(y_variance > 0.f))
        return rxg::fail(ctx, RXG_ERR_BAD_ARG, "hgf_filter: bad argument");
    if (!(flags & RXG_PTR_DEVICE)) return rxg::fail(ctx, RXG_ERR_UNSUPPORTED, "hgf_filter takes device pointers");
    RXG_CUDA(ctx, cudaSetDevice(ctx->device));
    int rc = ensure_gh_tables(ctx);
    if (rc != RXG_OK) return rc;
    const float z4[4] = {0.f, 1.f, 0.f, 1.f};
    const float* in = init ? init : z4;
    const unsigned grid = (unsigned)((batch + 63) / 64);
    if (free_energy)
        hgf_filter_kernel<true><<<grid, 64, 0, ctx->stream>>>(y, out, T, batch, iters, kappa, omega, z_variance, y_variance,
                                                             in[0], in[1], in[2], in[3], prev, free_energy);
    else
        hgf_filter_kernel<false><<<grid, 64, 0, ctx->stream>>>(y, out, T, batch, iters, kappa, omega, z_variance, y_variance,
                                                              in[0], in[1], in[2], in[3], prev, nullptr);
    ctx->launches += 1;
    rc = rxg::check_cuda(ctx, cudaGetLastError(), "hgf_filter_kernel");
    if (rc != RXG_OK) return rc;
    if (!(flags & RXG_ASYNC)) RXG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return RXG_OK;
}

int rxg_hgf_filter_f32(rxg_ctx* ctx, int T, int64_t batch, int iters, float kappa, float omega, float z_variance,
                       float y_variance, const float init[4], const float* y, float* out, unsigned flags) {
    if (ctx && !init) return rxg::fail(ctx, RXG_ERR_BAD_ARG, "hgf_filter: init is required");
    return rxg_hgf_filter_fe_f32(ctx, T, batch, iters, kappa, omega, z_variance, y_variance, init, nullptr, y, out, nullptr, flags);
}

int rxg_hgf_filter_chunk_f32(rxg_ctx* ctx, int T, int64_t batch, int iters, float kappa, float omega, float z_variance,
                             float y_variance, const float* prev, const float* y, float* out, unsigned flags) {
    if (ctx && !prev) return rxg::fail(ctx, RXG_ERR_BAD_ARG, "hgf_filter_chunk: prev is required");
    return rxg_hgf_filter_fe_f32(ctx, T, batch, iters, kappa, omega, z_variance, y_variance, nullptr, prev, y, out, nullptr, flags);
}

#define RXG_GCV_PROLOGUE                                                                          \
    if (!ctx) return RXG_ERR_BAD_ARG;                                                             \
    if (!(flags & RXG_PTR_DEVICE)) return rxg::fail(ctx, RXG_ERR_UNSUPPORTED, "GCV rules take device pointers"); \
    if (n <= 0) return n == 0 ? RXG_OK : rxg::fail(ctx, RXG_ERR_BAD_ARG, "n < 0");                \
    RXG_CUDA(ctx, cudaSetDevice(ctx->device));                                                    \
    { int rc0 = ensure_gh_tables(ctx); if (rc0 != RXG_OK) return rc0; }
#define RXG_GCV_EPILOGUE(what)                                                                    \
    ctx->launches += 1;                                                                           \
    { int rc1 = rxg::check_cuda(ctx, cudaGetLastError(), what); if (rc1 != RXG_OK) return rc1; }  \
    if (!(flags & RXG_ASYNC)) RXG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));                  \
    return RXG_OK;

int rxg_rule_gcv_out_f32(rxg_ctx* ctx, int64_t n, const float* m_x, const float* v_x, const float* m_z,
                         const float* v_z, float kappa, float omega, float* m_out, float* v_out, unsigned flags) {
    RXG_GCV_PROLOGUE
    k_gcv_out<<<(unsigned)((n + 255) / 256), 256, 0, ctx->stream>>>(n, m_x, v_x, m_z, v_z, kappa, omega, m_out, v_out);
    RXG_GCV_EPILOGUE("k_gcv_out")
}
int rxg_marginalrule_gcv_yx_f32(rxg_ctx* ctx, int64_t n, const float* m_y, const float* v_y, const float* m_x,
                                const float* v_x, const float* m_z, const float* v_z, float kappa, float omega,
                                float* m, float* V, unsigned flags) {
    RXG_GCV_PROLOGUE
    k_gcv_yx<<<(unsigned)((n + 255) / 256), 256, 0, ctx->stream>>>(n, m_y, v_y, m_x, v_x, m_z, v_z, kappa, omega, m, V);
    RXG_GCV_EPILOGUE("k_gcv_yx")
}
int rxg_rule_gcv_z_prod_f32(rxg_ctx* ctx, int64_t n, const float* m_yx, const float* V_yx, const float* m_zprior,
                            const float* v_zprior, float kappa, float omega, float* m_z, float* v_z,
                            unsigned flags) {
    RXG_GCV_PROLOGUE
    k_gcv_z_prod<<<(unsigned)((n + 127) / 128), 128, 0, ctx->stream>>>(n, m_yx, V_yx, m_zprior, v_zprior, kappa, omega, m_z, v_z);
    RXG_GCV_EPILOGUE("k_gcv_z_prod")
}

int rxg_lgssm_vmp_gamma_fe_f32(rxg_ctx* ctx, int T, int64_t batch, int iterations, float a, float v_proc, float m0,
                               float v0, float a0, float b0, float init_E_tau, const float* y, float* post_mean,
                               float* post_var, float* shape, float* rate, float* free_energy, unsigned flags);
int rxg_lgssm_vmp_gamma_f32(rxg_ctx* ctx, int T, int64_t batch, int iterations, float a, float v_proc, float m0,
                            float v0, float a0, float b0, float init_E_tau, const float* y, float* post_mean,
                            float* post_var, float* shape, float* rate, unsigned flags) {
    return rxg_lgssm_vmp_gamma_fe_f32(ctx, T, batch, iterations, a, v_proc, m0, v0, a0, b0, init_E_tau, y, post_mean, post_var,
                                      shape, rate, nullptr, flags);
}
int rxg_lgssm_vmp_gamma_fe_f32(rxg_ctx* ctx, int T, int64_t batch, int iterations, float a, float v_proc, float m0,
                               float v0, float a0, float b0, float init_E_tau, const float* y, float* post_mean,
                               float* post_var, float* shape, float* rate, float* free_energy, unsigned flags) {
    if (!ctx) return RXG_ERR_BAD_ARG;
    if (T < 1 || batch < 1 || iterations < 1 || !y || !post_mean || !post_var || !shape || !rate)
        return rxg::fail(ctx, RXG_ERR_BAD_ARG, "lgssm_vmp_gamma: bad argument");
    // variances, the Gamma prior and the initial E[tau] must be positive (NaN is refused too): lgammaf(a0), logf(b0), the
    // observation variance 1 / E[tau] and the RTS gain's division by the predicted variance need it
    if (!(v_proc > 0.f) || !(v0 > 0.f) || !(a0 > 0.f) || !(b0 > 0.f) || !(init_E_tau > 0.f))
        return rxg::fail(ctx, RXG_ERR_BAD_ARG, "lgssm_vmp_gamma: v_proc, v0, a0, b0 and init_E_tau must be positive");
    if (!(flags & RXG_PTR_DEVICE)) return rxg::fail(ctx, RXG_ERR_UNSUPPORTED, "lgssm_vmp_gamma takes device pointers");
    RXG_CUDA(ctx, cudaSetDevice(ctx->device));
    vmp_gamma_kernel<<<(unsigned)((batch + 127) / 128), 128, 0, ctx->stream>>>(
        y, post_mean, post_var, shape, rate, T, batch, iterations, a, v_proc, m0, v0, a0, b0, init_E_tau, free_energy);
    ctx->launches += 1;
    int rc = rxg::check_cuda(ctx, cudaGetLastError(), "vmp_gamma_kernel");
    if (rc != RXG_OK) return rc;
    if (!(flags & RXG_ASYNC)) RXG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return RXG_OK;
}

int rxg_stream_vmp_gamma_f32(rxg_ctx* ctx, int T, int64_t batch, int iters, float w, const float init[4],
                             const float* prev, const float* y, float* out, float* free_energy, unsigned flags) {
    if (!ctx) return RXG_ERR_BAD_ARG;
    if (T < 1 || batch < 1 || iters < 1 || !(w > 0.f) || !y || !out || (!init && !prev))
        return rxg::fail(ctx, RXG_ERR_BAD_ARG, "stream_vmp_gamma: bad argument");
    if (!(flags & RXG_PTR_DEVICE)) return rxg::fail(ctx, RXG_ERR_UNSUPPORTED, "stream_vmp_gamma takes device pointers");
    RXG_CUDA(ctx, cudaSetDevice(ctx->device));
    const float z[4] = {0.f, 1.f, 1.f, 1.f};
    const float* in = init ? init : z;
    stream_vmp_gamma_kernel<<<(unsigned)((batch + 127) / 128), 128, 0, ctx->stream>>>(
        y, prev, out, free_energy, T, batch, iters, w, in[0], in[1], in[2], in[3]);
    ctx->launches += 1;
    int rc = rxg::check_cuda(ctx, cudaGetLastError(), "stream_vmp_gamma_kernel");
    if (rc != RXG_OK) return rc;
    if (!(flags & RXG_ASYNC)) RXG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return RXG_OK;
}

}  // extern "C"
