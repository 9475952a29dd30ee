// Hierarchical Gaussian Filter with random coupling kappa and volatility offset omega, learned per series: naive
// mean-field VMP over the whole series, all iterations of one chain in one thread.
//
//     omega ~ N(m_w0, v_w0), kappa ~ N(m_k0, v_k0), x_0 ~ N(m_x0, v_x0), z_1 ~ N(m_z0, v_z0)
//     z_t ~ N(z_{t-1}, precision tau_z) (t >= 2);  x_t ~ GCV(x_{t-1}, z_t, kappa, omega);  y_t ~ N(x_t, v_y)
//     q = q(kappa) q(omega) q(x_0) prod_t q(x_t) q(z_t)
// [ref: model `hgf_1`, test/inference/inference_tests.jl:609-642, run with MeanField(); GCV average energy :587-607
//  (variance exp(kappa z + omega)); the five GCV rules it delegates to, :547-585].  DESIGN.md section 3.19.
//
// With A = exp(-m_w + v_w / 2), B_t = exp(-m_k m_zt + xi_t / 2), xi_t = m_k^2 v_zt + m_zt^2 v_k + v_k v_zt and
// psi_t = (m_xt - m_xt-1)^2 + v_xt + v_xt-1 the rules are
//   :x / :y   Gaussian messages of precision A B_t (q(x_t) is their exact product with the y message)
//   :z        ELQ(m_k, psi_t A, -m_k, v_k)        :kappa  ELQ(m_zt, psi_t A, -m_zt, v_zt)
//   :omega    ELQ(1, psi_t B_t, -1, 0)
// with ELQ(a, b, c, d)(u) = exp(-(a u + b exp(c u + d u^2 / 2)) / 2).  A Normal times an ELQ is GH-31 moment matching
// centred on the Normal (gh_prod).  Products fold left to right in node-creation order: q(z_t) = GH(message of the
// z_{t-1} node, ELQ_t) times the z_{t+1} node's message; q(kappa) = GH(...GH(GH(prior, ELQ_1), ELQ_2)..., ELQ_T) and
// q(omega) likewise, both refolded from the prior every iteration.
//
// One iteration is one Gauss-Seidel sweep: q(x_0), then for t = 1..T q(x_t) (new q(x_t-1), old q(x_t+1), q(z_t),
// q(z_t+1)), q(z_t) (new q(z_t-1), old q(z_t+1)), and ELQ_t folded into q(kappa) (old q(omega)) and q(omega) (old
// q(kappa)).  q(x_t), q(z_t) live in the output stash [T][4][batch] (m_x, v_x, m_z, v_z): a step reads the old marginals
// of t+1 and writes the new ones of t, 36 bytes with y.  The free energy of iteration i is summed in fp64 during sweep
// i + 1 from the old marginals before they are overwritten, and for the last iteration in one closing pass.
// A NaN y_t is a missing step (no y node).  A non-finite normaliser or result flags the chain RXG_ERR_NAN.
#pragma once
#include <math.h>
#include <stdint.h>

#ifndef RXG_HD
#define RXG_HD __host__ __device__ __forceinline__
#endif

namespace rxg {
namespace hgfl {

constexpr int NGH = 31;
constexpr int ST_NAN = 5;   // RXG_ERR_NAN

// Gauss-Hermite nodes (physicists' convention) and log2 of the weights, rounded to fp32, and vfix = 1 / (2 m2) with m2 the
// second moment sum_i w_i t_i^2 / sum_i w_i of the ROUNDED rule (exactly 1/2 for the exact one; the rounding moves it by
// ~4e-8).  A fold multiplies that bias into its variance once per step, 4e-4 after 10 000 steps, so each fold step
// divides it out (gh_fold).  fill_vfix sets it from t and lw2.
struct GH {
    float t[NGH];
    float lw2[NGH];
    double vfix;
};

inline void fill_vfix(GH& g) {
    double s0 = 0.0, s2 = 0.0;
    for (int i = 0; i < NGH; ++i) {
        const double w = exp2((double)g.lw2[i]), t = (double)g.t[i];
        s0 += w;
        s2 += w * t * t;
    }
    g.vfix = s0 / (2.0 * s2);
}

// per-launch hyper-parameters and initial marginals, shared by every chain
struct Prm {
    float mk0, vk0, mw0, vw0, mx0, vx0, mz0, vz0;   // priors of kappa, omega, x_0, z_1
    float tau_z, vy;                                // z transition precision, y variance
    float ik_m, ik_v, iw_m, iw_v;                   // initial q(kappa), q(omega)
    float iz_m, iz_v, ix_m, ix_v;                   // initial q(z_t), q(x_t), every t
};

struct Args {
    int T, iters;
    int64_t batch;
    Prm p;
    const float* y;    // [T][batch], NaN = missing
    float* x0;         // [2][batch]: q(x_0)
    float* xz;         // [T][4][batch]: q(x_t), q(z_t); also the stash
    float* kw;         // [2][2][batch]: (m, v) of q(kappa), then of q(omega)
    float* hist_kw;    // [iters][2][2][batch] or null
    double* fe;        // [iters][batch] or null
};

struct N1 {
    float m, v;
};

// a fold's running Normal: the mean in fp64, so that a thousand small shifts are not each rounded onto an O(1) fp32 mean;
// the variance is updated in fp64 (with the bias correction GH::vfix, which fp32 would round to 1) and stored in fp32
struct Fold {
    double m;
    float v;
};

RXG_HD float ex2(float x) {
#ifdef __CUDA_ARCH__
    float r;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
    return r;
#else
    return exp2f(x);
#endif
}

RXG_HD bool finite_pos(float v) { return v > 0.f && v <= 3.402823466e38f; }

// prod(N(mu, v), ELQ(a, b, c, d)) by GH-31 moment matching centred on the Normal: nodes z_i = mu + u_i, u_i = sqrt(2 v) t_i,
// log2 weights lw2_i - log2(e) / 2 (a u_i + b exp(c z_i + d z_i^2 / 2)) (the a mu term is common to all nodes), the
// variance taken about the new mean (fp32: in a third pass).  Returns the mean shift du = E[t] and the variance ratio
// rho = 2 Var[t] in units of the nodes t_i (new variance = v rho); flags st on a non-finite normaliser or result.
// Acc is the type of the moment sums: fp32 for the z products, fp64 for the folds, where T nearly identical products in a
// row would otherwise repeat the same fp32 rounding of the sums T times.
template <typename Acc>
struct Moments {
    Acc dt, rho;
};

template <typename Acc>
RXG_HD Moments<Acc> gh_moments(const GH& gh, float mu, float s, float a, float b, float c, float d, int& st) {
    constexpr float L2E = 1.4426950408889634f;
    const float ha = -0.5f * L2E * a, hb = -0.5f * L2E * b, c2 = L2E * c, d2 = 0.5f * L2E * d;
    float l[NGH];
    float lmax = -INFINITY;
#pragma unroll
    for (int i = 0; i < NGH; ++i) {
        const float u = s * gh.t[i];
        const float z = mu + u;
        l[i] = fmaf(hb, ex2(z * fmaf(d2, z, c2)), fmaf(ha, u, gh.lw2[i]));
        lmax = fmaxf(lmax, l[i]);
    }
    Acc S0 = 0, S1 = 0, S2 = 0;
    if constexpr (sizeof(Acc) == sizeof(double)) {   // fp64: E[t^2] - E[t]^2 has no cancellation to fear, one pass
#pragma unroll
        for (int i = 0; i < NGH; ++i) {
            const double e = ex2(l[i] - lmax), t = gh.t[i];
            S0 += e;
            S1 = fma(e, t, S1);
            S2 = fma(e * t, t, S2);
        }
    } else {                                         // fp32: the variance about the new mean in a third pass
#pragma unroll
        for (int i = 0; i < NGH; ++i) {
            l[i] = ex2(l[i] - lmax);
            S0 += l[i];
            S1 = fmaf(l[i], gh.t[i], S1);
        }
    }
    const Acc r = (Acc)1 / S0;
    const Acc dt = S1 * r;
    if constexpr (sizeof(Acc) == sizeof(double)) {
        S2 = fma(-dt, dt, S2 * r) * S0;
    } else {
#pragma unroll
        for (int i = 0; i < NGH; ++i) {
            const float w = gh.t[i] - dt;
            S2 = fmaf(l[i] * w, w, S2);
        }
    }
    const Moments<Acc> q{dt, 2 * S2 * r};
    if (!finite_pos((float)S0) || !(fabsf(mu + s * (float)dt) <= 3.402823466e38f) || !finite_pos((float)q.rho) ||
        !finite_pos(s))
        st = ST_NAN;
    return q;
}

RXG_HD N1 gh_prod(const GH& gh, float mu, float v, float a, float b, float c, float d, int& st) {
    const float s = sqrtf(2.f * v);
    const Moments<float> q = gh_moments<float>(gh, mu, s, a, b, c, d, st);
    return {fmaf(s, q.dt, mu), v * q.rho};
}

RXG_HD void gh_fold(const GH& gh, Fold& f, float a, float b, float c, float d, int& st) {
    const float s = sqrtf(2.f * f.v);
    const Moments<double> q = gh_moments<double>(gh, (float)f.m, s, a, b, c, d, st);
    f.m = fma((double)s, q.dt, f.m);
    f.v = (float)((double)f.v * q.rho * gh.vfix);
}

// B = exp(-m_k m_z + xi / 2), xi = m_k^2 v_z + m_z^2 v_k + v_k v_z  [ref: inference_tests.jl:601-604]
RXG_HD float gcv_B(float mk, float vk, float mz, float vz) {
    const float xi = fmaf(mk * mk, vz, fmaf(mz * mz, vk, vk * vz));
    return expf(fmaf(0.5f, xi, -mk * mz));
}

constexpr float LOG_2PI = 1.8378770664093453f;

// E_q[-log N(u; m0, v0)] of a Normal prior at q(u) = N(m, v)
RXG_HD float prior_energy(float m, float v, float m0, float v0) {
    const float d = m - m0;
    return 0.5f * (LOG_2PI + logf(v0) + fmaf(d, d, v) / v0);
}

RXG_HD float entropy(float v) { return 0.5f * (LOG_2PI + 1.f + logf(v)); }

// The free-energy terms of step t (1-based t = 1 for `first`) from the marginals q(x_t-1), q(x_t), q(z_t-1), q(z_t) and
// q(kappa), q(omega): the GCV node (:606 verbatim), the z prior or transition, the y node if observed, minus the
// entropies of x_t and z_t.
RXG_HD float step_energy(const Prm& p, N1 xp, N1 x, N1 zp, N1 z, bool first, float yt, float mk, float vk, float mw,
                         float vw) {
    const float dx = x.m - xp.m;
    const float psi = fmaf(dx, dx, x.v + xp.v);
    const float A = expf(fmaf(0.5f, vw, -mw));
    float U = 0.5f * (LOG_2PI + fmaf(z.m, mk, mw) + psi * A * gcv_B(mk, vk, z.m, z.v));
    if (first) {
        U += prior_energy(z.m, z.v, p.mz0, p.vz0);
    } else {
        const float dz = z.m - zp.m;
        U += 0.5f * (LOG_2PI - logf(p.tau_z) + p.tau_z * fmaf(dz, dz, z.v + zp.v));
    }
    if (yt == yt) U += prior_energy(x.m, x.v, yt, p.vy);
    return U - entropy(x.v) - entropy(z.v);
}

// the terms outside the steps: priors and entropies of kappa, omega and x_0
RXG_HD double global_energy(const Prm& p, N1 x0, float mk, float vk, float mw, float vw) {
    return (double)(prior_energy(mk, vk, p.mk0, p.vk0) - entropy(vk)) +
           (double)(prior_energy(mw, vw, p.mw0, p.vw0) - entropy(vw)) +
           (double)(prior_energy(x0.m, x0.v, p.mx0, p.vx0) - entropy(x0.v));
}

// One chain.  Returns its status (0 or ST_NAN).
template <bool FE>
RXG_HD int chain(int64_t b, const Args& a, const GH& gh) {
    const Prm& p = a.p;
    const int T = a.T;
    const int64_t nb = a.batch;
    float* xz = a.xz;
    const float* y = a.y;
    auto at = [&](int t, int r) { return ((int64_t)t * 4 + r) * nb + b; };
    const float vzt = 1.f / p.tau_z, wy = 1.f / p.vy;
    int st = 0;
    float mk = p.ik_m, vk = p.ik_v, mw = p.iw_m, vw = p.iw_v;
    N1 x0{p.mx0, p.vx0};
    for (int it = 0; it < a.iters; ++it) {
        const bool fresh = it == 0;   // the stash holds nothing yet: the old q(x_t), q(z_t) are the initialisation
        const bool fe_prev = FE && !fresh;
        const float A = expf(fmaf(0.5f, vw, -mw));
        N1 ox{p.ix_m, p.ix_v}, oz{p.iz_m, p.iz_v};   // old q(x_t), q(z_t) of the current step
        if (!fresh) { ox = {xz[at(0, 0)], xz[at(0, 1)]}; oz = {xz[at(0, 2)], xz[at(0, 3)]}; }
        // q(x_0) = prior x GCV_1's message N(m_x1, 1 / (A B_1))
        const N1 ox0 = x0;
        {
            const float g = A * gcv_B(mk, vk, oz.m, oz.v);
            const float w = 1.f / p.vx0 + g;
            x0.v = 1.f / w;
            x0.m = x0.v * fmaf(g, ox.m, p.mx0 / p.vx0);
        }
        double F = fe_prev ? global_energy(p, ox0, mk, vk, mw, vw) : 0.0;
        N1 xp = x0;                    // new q(x_t-1)
        float mzp = 0.f;               // new m_z of t-1
        N1 pox = ox0, poz{0.f, 1.f};   // old q(x_t-1), q(z_t-1) (free energy of the previous iteration)
        Fold fk{p.mk0, p.vk0}, fw{p.mw0, p.vw0};
        float ynext = y[b];
        for (int t = 0; t < T; ++t) {
            const float yt = ynext;
            const bool more = t + 1 < T;
            N1 nx{p.ix_m, p.ix_v}, nz{p.iz_m, p.iz_v};   // old q(x_t+1), q(z_t+1)
            if (more) {
                ynext = y[(int64_t)(t + 1) * nb + b];
                if (!fresh) { nx = {xz[at(t + 1, 0)], xz[at(t + 1, 1)]}; nz = {xz[at(t + 1, 2)], xz[at(t + 1, 3)]}; }
            }
            const bool obs = yt == yt;
            // q(x_t): GCV_t message N(m_xt-1, 1 / g_t), GCV_t+1 message N(m_xt+1, 1 / g_n), y message N(y_t, v_y)
            const float g = A * gcv_B(mk, vk, oz.m, oz.v);
            const float gn = more ? A * gcv_B(mk, vk, nz.m, nz.v) : 0.f;
            const float w = g + gn + (obs ? wy : 0.f);
            N1 x;
            x.v = 1.f / w;
            x.m = x.v * fmaf(g, xp.m, fmaf(gn, more ? nx.m : 0.f, obs ? yt * wy : 0.f));
            const float dx = x.m - xp.m;
            const float psi = fmaf(dx, dx, x.v + xp.v);
            // q(z_t) = GH(z_t-1 node's message, ELQ_t) x z_t+1 node's message
            N1 z = t == 0 ? gh_prod(gh, p.mz0, p.vz0, mk, psi * A, -mk, vk, st)
                          : gh_prod(gh, mzp, vzt, mk, psi * A, -mk, vk, st);
            if (more) {
                const float wz = 1.f / z.v + p.tau_z;
                const float v = 1.f / wz;
                z.m = v * fmaf(nz.m, p.tau_z, z.m / z.v);
                z.v = v;
            }
            if (fe_prev) F += (double)step_energy(p, pox, ox, poz, oz, t == 0, yt, mk, vk, mw, vw);
            // ELQ_t folded into q(kappa) (with the old q(omega)) and q(omega) (with the old q(kappa))
            gh_fold(gh, fk, z.m, psi * A, -z.m, z.v, st);
            gh_fold(gh, fw, 1.f, psi * gcv_B(mk, vk, z.m, z.v), -1.f, 0.f, st);
            xz[at(t, 0)] = x.m;
            xz[at(t, 1)] = x.v;
            xz[at(t, 2)] = z.m;
            xz[at(t, 3)] = z.v;
            pox = ox; poz = oz; ox = nx; oz = nz;
            xp = x; mzp = z.m;
        }
        if (fe_prev) a.fe[(int64_t)(it - 1) * nb + b] = F;
        mk = (float)fk.m; vk = fk.v; mw = (float)fw.m; vw = fw.v;
        if (a.hist_kw) {
            float* h = a.hist_kw + (int64_t)it * 4 * nb + b;
            h[0] = mk; h[nb] = vk; h[2 * nb] = mw; h[3 * nb] = vw;
        }
    }
    if (FE) {   // closing pass: the free energy of the last iteration from the stash
        double F = global_energy(p, x0, mk, vk, mw, vw);
        N1 xp = x0, zp{0.f, 1.f};
        for (int t = 0; t < T; ++t) {
            const N1 x{xz[at(t, 0)], xz[at(t, 1)]}, z{xz[at(t, 2)], xz[at(t, 3)]};
            F += (double)step_energy(p, xp, x, zp, z, t == 0, y[(int64_t)t * nb + b], mk, vk, mw, vw);
            xp = x; zp = z;
        }
        a.fe[(int64_t)(a.iters - 1) * nb + b] = F;
    }
    if (a.x0) { a.x0[b] = x0.m; a.x0[nb + b] = x0.v; }
    a.kw[b] = mk; a.kw[nb + b] = vk; a.kw[2 * nb + b] = mw; a.kw[3 * nb + b] = vw;
    return st;
}

}  // namespace hgfl
}  // namespace rxg
