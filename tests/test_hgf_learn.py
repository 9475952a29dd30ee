"""The HGF with learned coupling kappa and volatility offset omega (RxInfer test/inference/inference_tests.jl:609-642,
`hgf_1` under MeanField()), on the CPU.

This module holds the fp64 reference the CUDA kernel (csrc/rxg_hgf_learn.cuh) is gated against, as test_hmm.py does for
the hidden Markov model:
  omega ~ N(m_w0, v_w0), kappa ~ N(m_k0, v_k0), x_0 ~ N(m_x0, v_x0), z_1 ~ N(m_z0, v_z0)
  z_t ~ N(z_{t-1}, precision tau_z);  x_t ~ GCV(x_{t-1}, z_t, kappa, omega) (variance exp(kappa z_t + omega));
  y_t ~ N(x_t, v_y);  q(kappa) q(omega) q(x_0) prod_t q(x_t) q(z_t)
One iteration is one Gauss-Seidel sweep over t (DESIGN 3.19).  The checks here: every update against an independent
computation (a dense Gaussian product, quadrature of the Normal x ELQ integrand, repeated single products for the folds),
the free energy against a term-by-term restatement, the fixed-parameter limit, the reference test's configuration,
recovery of kappa and omega from simulated series, the kernel body compiled for the host
(tests/c/hgf_learn_host_harness.cu), and the host-side argument handling."""
import ctypes
import os
import shutil
import subprocess
import tempfile

import numpy as np
import pytest
from scipy import integrate, stats
from scipy.special import roots_hermite

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LOG_2PI = np.log(2 * np.pi)

# (m, v) of kappa, omega, x_0, z_1 -- the reference's priors (:610-613) -- then tau_z, v_y, and the initial q(kappa),
# q(omega), q(z), q(x) of :624-629
DEFAULT = dict(prior=(1.0, 1.0, 0.0, 1.0, 0.0, 1.0, 0.0, 1.0), z_precision=1.0, y_variance=1.0,
               init=(1.0, 1.0, 0.0, 1.0, 0.0, 1.0, 0.0, 1.0))
# two non-default sets, no value equal to 0 or 1
SET_B = dict(prior=(0.7, 0.3, -0.4, 0.5, 0.2, 2.0, -0.3, 0.6), z_precision=2.5, y_variance=0.3,
             init=(0.8, 0.4, -0.2, 0.6, 0.1, 0.7, 0.3, 1.5))
SET_C = dict(prior=(1.3, 0.2, 0.5, 0.25, -0.5, 0.5, 0.4, 1.5), z_precision=4.0, y_variance=0.05,
             init=(1.2, 0.3, 0.4, 0.3, -0.2, 2.0, -0.1, 0.8))
HYPER = {"default": DEFAULT, "B": SET_B, "C": SET_C}


# --------------------------------------------------------------------------- fp64 reference
def gh_nodes():
    return roots_hermite(31)


def gh_prod(n, elq, nw=None):
    """prod(N(m, v), ELQ(a, b, c, d)) by GH-31 moment matching centred on the Normal (log-domain weights)."""
    t, w = nw if nw is not None else gh_nodes()
    m, v = (np.asarray(u, np.float64) for u in n)
    a, b, c, d = (np.asarray(u, np.float64)[..., None] for u in elq)
    z = m[..., None] + np.sqrt(2.0 * v)[..., None] * t
    l = np.log(w) - 0.5 * (a * (z - m[..., None]) + b * np.exp(c * z + 0.5 * d * z * z))
    e = np.exp(l - l.max(-1, keepdims=True))
    Z = e.sum(-1)
    mz = (e * z).sum(-1) / Z
    return mz, (e * (z - mz[..., None]) ** 2).sum(-1) / Z


def gcv_B(mk, vk, mz, vz):
    """B = exp(-m_k m_z + xi / 2), xi = m_k^2 v_z + m_z^2 v_k + v_k v_z (inference_tests.jl:601-604)."""
    return np.exp(-mk * mz + 0.5 * (mk * mk * vz + mz * mz * vk + vk * vz))


def x_update(xp, xn, g, gn, y, v_y):
    """q(x_t): product of the GCV_t message N(m_xt-1, 1/g), the GCV_t+1 message N(m_xt+1, 1/gn) (gn = 0: none) and the
    y message N(y, v_y) (y NaN: none), in precision form."""
    obs = ~np.isnan(y)
    wy = np.where(obs, 1.0 / v_y, 0.0)
    w = g + gn + wy
    return (g * xp + gn * xn + np.where(obs, y, 0.0) * wy) / w, 1.0 / w


def hgf_learn(y, iterations, prior, z_precision, y_variance, init, learn=True):
    """The kernel's schedule in fp64.  y[T, batch] (NaN = missing).  learn=False holds kappa, omega at the prior means as
    point masses.  Returns x0[2, b], xz[T, 4, b], kw[2, 2, b], hist_kw[its, 2, 2, b], free_energy[its, b]."""
    y = np.asarray(y, np.float64)
    T, nb = y.shape
    nw = gh_nodes()
    mk0, vk0, mw0, vw0, mx0, vx0, mz0, vz0 = prior
    full = lambda v: np.full(nb, float(v))
    if learn:
        mk, vk, mw, vw = full(init[0]), full(init[1]), full(init[2]), full(init[3])
    else:
        mk, vk, mw, vw = full(mk0), full(0.0), full(mw0), full(0.0)
    zm, zv = np.full((T, nb), float(init[4])), np.full((T, nb), float(init[5]))
    xm, xv = np.full((T, nb), float(init[6])), np.full((T, nb), float(init[7]))
    vzt = 1.0 / z_precision
    hist, fes = [], []
    min_vz = np.full(nb, np.inf)          # the smallest q(z_t) variance any update produced
    for _ in range(iterations):
        A = np.exp(-mw + 0.5 * vw)
        g1 = A * gcv_B(mk, vk, zm[0], zv[0])
        x0v = 1.0 / (1.0 / vx0 + g1)
        x0m = x0v * (mx0 / vx0 + g1 * xm[0])
        fk, fw = (full(mk0), full(vk0)), (full(mw0), full(vw0))
        mxp, vxp = x0m, x0v
        for t in range(T):
            more = t + 1 < T
            g = A * gcv_B(mk, vk, zm[t], zv[t])
            gn = A * gcv_B(mk, vk, zm[t + 1], zv[t + 1]) if more else 0.0
            xm[t], xv[t] = x_update(mxp, xm[t + 1] if more else 0.0, g, gn, y[t], y_variance)
            psi = (xm[t] - mxp) ** 2 + xv[t] + vxp
            src = (full(mz0), full(vz0)) if t == 0 else (zm[t - 1], full(vzt))
            m1, v1 = gh_prod(src, (mk, psi * A, -mk, vk), nw)
            if more:
                w = 1.0 / v1 + z_precision
                m1, v1 = (m1 / v1 + zm[t + 1] * z_precision) / w, 1.0 / w
            zm[t], zv[t] = m1, v1
            min_vz = np.fmin(min_vz, v1)
            if learn:
                fk = gh_prod(fk, (zm[t], psi * A, -zm[t], zv[t]), nw)
                fw = gh_prod(fw, (np.ones(nb), psi * gcv_B(mk, vk, zm[t], zv[t]), -np.ones(nb), np.zeros(nb)), nw)
            mxp, vxp = xm[t], xv[t]
        if learn:
            (mk, vk), (mw, vw) = fk, fw
        hist.append(np.stack([np.stack([mk, vk]), np.stack([mw, vw])]))
        if learn:
            fes.append(free_energy(y, (x0m, x0v), xm, xv, zm, zv, (mk, vk), (mw, vw), prior, z_precision, y_variance))
    return dict(x0=np.stack([x0m, x0v]), xz=np.stack([xm, xv, zm, zv], 1), kw=hist[-1], hist_kw=np.stack(hist),
                free_energy=np.stack(fes) if learn else None, min_vz=min_vz)


def free_energy(y, x0, xm, xv, zm, zv, qk, qw, prior, z_precision, y_variance):
    """Mean-field VMP free energy: sum over nodes of E_q[-log f] minus the sum over variables of H[q]."""
    mk0, vk0, mw0, vw0, mx0, vx0, mz0, vz0 = prior
    (mk, vk), (mw, vw) = qk, qw
    nrg = lambda m, v, m0, v0: 0.5 * (LOG_2PI + np.log(v0) + ((m - m0) ** 2 + v) / v0)
    ent = lambda v: 0.5 * (LOG_2PI + 1.0 + np.log(v))
    F = nrg(mk, vk, mk0, vk0) + nrg(mw, vw, mw0, vw0) + nrg(x0[0], x0[1], mx0, vx0) + nrg(zm[0], zv[0], mz0, vz0)
    pm = np.concatenate([x0[0][None], xm[:-1]])
    pv = np.concatenate([x0[1][None], xv[:-1]])
    psi = (xm - pm) ** 2 + xv + pv
    A = np.exp(-mw + 0.5 * vw)
    F = F + (0.5 * (LOG_2PI + (zm * mk + mw) + psi * A * gcv_B(mk, vk, zm, zv))).sum(0)
    F = F + (0.5 * (LOG_2PI - np.log(z_precision) + z_precision * ((zm[1:] - zm[:-1]) ** 2 + zv[1:] + zv[:-1]))).sum(0)
    obs = ~np.isnan(y)
    F = F + np.where(obs, nrg(xm, xv, np.where(obs, y, 0.0), y_variance), 0.0).sum(0)
    return F - ent(vk) - ent(vw) - ent(x0[1]) - ent(xv).sum(0) - ent(zv).sum(0)


def f32(h):
    """The hyper-parameters as the ABI sees them: rounded to fp32 once."""
    return dict(prior=tuple(np.float32(h["prior"]).astype(float)), z_precision=float(np.float32(h["z_precision"])),
                y_variance=float(np.float32(h["y_variance"])), init=tuple(np.float32(h["init"]).astype(float)))


def series(T, nb, seed, kappa=0.8, omega=-0.5, p_missing=0.0):
    """Series drawn from the model (oracle/hgf.py generate_data) with a share of missing steps."""
    from oracle.hgf import generate_data
    _, _, y = generate_data(T, nb, kappa=kappa, omega=omega, z_variance=0.01, y_variance=0.2, seed=seed)
    y = y.astype(np.float64)
    if p_missing:
        y[np.random.default_rng(seed + 1).random(y.shape) < p_missing] = np.nan
    return y


# --------------------------------------------------------------------------- single updates
def test_x_update_is_the_dense_gaussian_product():
    rng = np.random.default_rng(1)
    grid = np.linspace(-30, 30, 600001)
    for _ in range(5):
        xp, xn, y = rng.normal(size=3)
        g, gn, vy = rng.uniform(0.2, 3.0, size=3)
        for obs in (True, False):
            yy = y if obs else np.nan
            m, v = x_update(np.array(xp), np.array(xn), g, gn, np.array(yy), vy)
            dens = stats.norm.pdf(grid, xp, np.sqrt(1 / g)) * stats.norm.pdf(grid, xn, np.sqrt(1 / gn))
            if obs:
                dens = dens * stats.norm.pdf(grid, y, np.sqrt(vy))
            dens /= np.trapezoid(dens, grid)
            md = np.trapezoid(grid * dens, grid)
            vd = np.trapezoid((grid - md) ** 2 * dens, grid)
            assert abs(m - md) < 1e-8 and abs(v - vd) < 1e-8


@pytest.mark.parametrize("elq", [(1.0, 0.7, -1.0, 0.0), (0.8, 1.3, -0.8, 0.3), (-0.4, 0.5, 0.6, 0.2), (1.5, 2.0, -1.2, 0.05)])
def test_gh_product_matches_quadrature(elq):
    """Normal x ELQ by GH-31 against scipy quad of the same integrand, where GH-31 is accurate (a Normal of moderate
    width, an ELQ that is smooth over it).  Also the same as oracle/rules.py's product (d = 0 there) where it applies."""
    from oracle import rules as R
    for m0, v0 in ((0.3, 0.5), (-0.2, 0.2), (1.0, 1.0)):
        a, b, c, d = elq
        f = lambda u, k: u ** k * stats.norm.pdf(u, m0, np.sqrt(v0)) * np.exp(-0.5 * (a * u + b * np.exp(c * u + 0.5 * d * u * u)))
        lo, hi = m0 - 12 * np.sqrt(v0), m0 + 12 * np.sqrt(v0)
        Z = integrate.quad(f, lo, hi, args=(0,), epsabs=0, epsrel=1e-13)[0]
        mq = integrate.quad(f, lo, hi, args=(1,), epsabs=0, epsrel=1e-13)[0] / Z
        vq = integrate.quad(lambda u: (u - mq) ** 2 * f(u, 0), lo, hi, epsabs=0, epsrel=1e-13)[0] / Z
        m, v = gh_prod((np.array(m0), np.array(v0)), elq)
        assert abs(m - mq) < 1e-5 * max(1, abs(mq)) and abs(v - vq) < 1e-5 * vq, (elq, m0, v0, m - mq, v / vq - 1)
        mr, vr = R.prod_normal_elq((np.array(m0), np.array(v0)), elq)
        assert abs(m - mr) < 1e-12 and abs(v - vr) < 1e-12


def test_folds_are_repeated_single_products():
    """After one sweep from the initialisation, q(kappa) and q(omega) are the prior folded with ELQ_1 .. ELQ_T one product
    at a time, each ELQ rebuilt from the final q(x_t), q(z_t) of that sweep and the initial q(kappa), q(omega) -- with
    oracle/rules.py's independent product."""
    from oracle import rules as R
    h = SET_B
    y = series(40, 3, seed=5, p_missing=0.2)
    r = hgf_learn(y, 1, **h)
    mk0, vk0, mw0, vw0 = h["prior"][:4]
    ik, ikv, iw, iwv = h["init"][:4]
    xm, xv, zm, zv = r["xz"][:, 0], r["xz"][:, 1], r["xz"][:, 2], r["xz"][:, 3]
    pm = np.concatenate([r["x0"][0][None], xm[:-1]])
    pv = np.concatenate([r["x0"][1][None], xv[:-1]])
    psi = (xm - pm) ** 2 + xv + pv
    A = np.exp(-iw + 0.5 * iwv)
    qk = (np.full(3, mk0), np.full(3, vk0))
    qw = (np.full(3, mw0), np.full(3, vw0))
    for t in range(40):
        qk = R.prod_normal_elq(qk, (zm[t][:, None], psi[t] * A, -zm[t][:, None], zv[t][:, None]))
        qw = R.prod_normal_elq(qw, (1.0, psi[t] * gcv_B(ik, ikv, zm[t], zv[t]), -1.0, 0.0))
    np.testing.assert_allclose(r["kw"][0], np.stack(qk), rtol=1e-10)
    np.testing.assert_allclose(r["kw"][1], np.stack(qw), rtol=1e-10)


def test_free_energy_term_by_term():
    """F against its definition restated term by term: scipy entropies, the Normal node energies by quadrature, the GCV
    energy exactly as inference_tests.jl:606."""
    h = SET_C
    y = series(6, 2, seed=3)
    y[2, 1] = np.nan
    r = hgf_learn(y, 3, **h)
    mk0, vk0, mw0, vw0, mx0, vx0, mz0, vz0 = h["prior"]
    tau, vy = h["z_precision"], h["y_variance"]
    for b in range(2):
        (mk, vk), (mw, vw) = r["kw"][0][:, b], r["kw"][1][:, b]
        x0m, x0v = r["x0"][:, b]
        xm, xv, zm, zv = (r["xz"][:, i, b] for i in range(4))

        def node(m, v, f):            # E_{N(m, v)}[f] by quadrature
            return integrate.quad(lambda u: stats.norm.pdf(u, m, np.sqrt(v)) * f(u), m - 15 * np.sqrt(v), m + 15 * np.sqrt(v),
                                  epsabs=0, epsrel=1e-12)[0]

        def pair(m1, v1, m2, v2, f):  # E over two independent Normals
            return integrate.quad(lambda u: stats.norm.pdf(u, m1, np.sqrt(v1)) * node(m2, v2, lambda w: f(u, w)),
                                  m1 - 12 * np.sqrt(v1), m1 + 12 * np.sqrt(v1), epsabs=0, epsrel=1e-10)[0]

        nlp = lambda m0, v0: (lambda u: -stats.norm.logpdf(u, m0, np.sqrt(v0)))
        U = node(mk, vk, nlp(mk0, vk0)) + node(mw, vw, nlp(mw0, vw0)) + node(x0m, x0v, nlp(mx0, vx0)) + node(zm[0], zv[0], nlp(mz0, vz0))
        pm, pv = np.concatenate([[x0m], xm[:-1]]), np.concatenate([[x0v], xv[:-1]])
        for t in range(6):
            ksi = mk ** 2 * zv[t] + zm[t] ** 2 * vk + vk * zv[t]
            psi = (xm[t] - pm[t]) ** 2 + xv[t] + pv[t]
            U += (LOG_2PI + (zm[t] * mk + mw) + psi * np.exp(-mw + vw / 2) * np.exp(-mk * zm[t] + ksi / 2)) / 2
            if t > 0:
                U += pair(zm[t], zv[t], zm[t - 1], zv[t - 1], lambda u, w: -stats.norm.logpdf(u, w, np.sqrt(1 / tau)))
            if not np.isnan(y[t, b]):
                U += node(xm[t], xv[t], lambda u: -stats.norm.logpdf(y[t, b], u, np.sqrt(vy)))
        H = sum(stats.norm(0, np.sqrt(v)).entropy() for v in [vk, vw, x0v, *xv, *zv])
        assert abs((U - H) - r["free_energy"][-1, b]) < 1e-8 * max(1, abs(U - H))


def test_tiny_prior_variances_reduce_to_fixed_parameters():
    """Prior (and initial) variances of kappa and omega at 1e-12: q(kappa), q(omega) stay at the prior, and q(x), q(z)
    match the same reference run with kappa, omega held as point masses."""
    y = series(50, 4, seed=11, p_missing=0.1)
    h = dict(SET_B)
    pr, ini = list(h["prior"]), list(h["init"])
    pr[1] = pr[3] = 1e-12
    ini[0], ini[1], ini[2], ini[3] = pr[0], 1e-12, pr[2], 1e-12
    h = dict(h, prior=tuple(pr), init=tuple(ini))
    r = hgf_learn(y, 5, **h)
    fixed = hgf_learn(y, 5, **h, learn=False)
    np.testing.assert_allclose(r["kw"][:, 0], [[pr[0]] * 4, [pr[2]] * 4], atol=1e-9)
    np.testing.assert_allclose(r["kw"][:, 1], 1e-12, rtol=1e-6)
    np.testing.assert_allclose(r["xz"], fixed["xz"], rtol=1e-8, atol=1e-9)
    np.testing.assert_allclose(r["x0"], fixed["x0"], rtol=1e-8, atol=1e-9)


# The largest increase of F between consecutive iterations over the checks below (the reference asserts a non-increasing
# F, inference_tests.jl:642, but its run has one iteration; GH moment matching is not the Gaussian-family optimum and the
# :606 energy uses the approximate B).  Measured with this reference, recorded in DESIGN 3.19.
def reference_data():
    """The `hgf_1` configuration: T = 6, y ~ N(0, 1) (seeded; the reference draws `rand(NormalMeanVariance(0, 1), 6)`)."""
    return np.random.default_rng(2024).standard_normal((6, 1))


def hgf1_assertions(x_mean, x_var, fe):
    """The reference's assertions on q(x) (:640-641), and what holds of F over 10 iterations: it decreases over the first
    six (by 1.0 at the first step), then rises by at most 2.5e-3 per iteration (2.46e-3 in the fp64 reference) as the GH
    fixed point settles.  The reference's `all(diff(F) .<= 0)` (:642) is vacuous for its single iteration."""
    assert np.all(~np.isnan(x_mean)) and np.all(~np.isnan(x_var))
    assert np.all(np.isfinite(fe)) and fe.shape[0] == 10
    d = np.diff(fe, axis=0)
    assert np.all(d[:5] < 0), d
    assert d.max() < 2.5e-3, d


def test_reference_configuration():
    y = reference_data()
    r = hgf_learn(y, 10, **DEFAULT)
    hgf1_assertions(r["xz"][:, 0], r["xz"][:, 1], r["free_energy"])


@pytest.mark.xfail(strict=True, reason="finding: on these series the mean-field fit drives E[kappa] to 4-6 (true 0.5-1.5) and "
                                      "19 of 256 chains end in a collapsed GH product (DESIGN 3.19)")
def test_recovers_kappa_and_omega_from_simulated_series():
    """256 series of 1000 steps drawn from the model at 16 (kappa, omega) pairs: the mean absolute error of E[kappa] and
    E[omega] after 20 iterations is below the prior mean's.  It is not, with this reading of the reference's rules: kept
    as a strict xfail so that the finding stays visible and a fix shows up."""
    from oracle.hgf import generate_data
    rng = np.random.default_rng(7)
    kappas, omegas = rng.uniform(0.5, 1.5, 16), rng.uniform(-1.0, 1.0, 16)
    zvar, yvar = 0.04, 0.01
    ys = [generate_data(1000, 16, kappa=k, omega=w, z_variance=zvar, y_variance=yvar, seed=100 + i)[2]
          for i, (k, w) in enumerate(zip(kappas, omegas))]
    y = np.concatenate(ys, axis=1).astype(np.float64)
    tk, tw = np.repeat(kappas, 16), np.repeat(omegas, 16)
    h = dict(prior=(1.0, 1.0, 0.0, 1.0, 0.0, 1.0, 0.0, zvar), z_precision=1 / zvar, y_variance=yvar,
             init=(1.0, 1.0, 0.0, 1.0, 0.0, zvar, 0.0, 1.0))
    r = hgf_learn(y, 20, **h)
    ek, ew = np.abs(r["kw"][0, 0] - tk).mean(), np.abs(r["kw"][1, 0] - tw).mean()
    pk, pw = np.abs(1.0 - tk).mean(), np.abs(0.0 - tw).mean()
    assert ek < pk and ew < pw, (ek, pk, ew, pw)


# --------------------------------------------------------------------------- the kernel body compiled for the host
_HARNESS = {}


def _host_harness():
    if "lib" in _HARNESS:
        return _HARNESS["lib"]
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    so = os.path.join(tempfile.mkdtemp(prefix="hgf_learn_host_"), "hgf_learn_host.so")
    src = os.path.join(ROOT, "tests", "c", "hgf_learn_host_harness.cu")
    subprocess.run([nvcc, "-O2", "-Wno-deprecated-gpu-targets", "-shared", "-Xcompiler", "-fPIC", "-o", so, src], check=True)
    _HARNESS["lib"] = ctypes.CDLL(so)
    return _HARNESS["lib"]


def gh_tables():
    t, w = gh_nodes()
    return np.float32(t), np.float32(np.log2(w))


def run_host(lib, y, iterations, prior, z_precision, y_variance, init, want_free_energy=True):
    T, nb = y.shape
    z = lambda *s: np.zeros(s, np.float32)
    out = dict(x0=z(2, nb), xz=z(T, 4, nb), kw=z(2, 2, nb), hist_kw=z(iterations, 2, 2, nb),
               free_energy=np.zeros((iterations, nb)) if want_free_energy else None, status=np.zeros(nb, np.int32))
    P = lambda a: None if a is None else a.ctypes.data_as(ctypes.c_void_p)
    t, lw2 = gh_tables()
    yy = np.ascontiguousarray(y, np.float32)
    pr, ini = np.float32(prior), np.float32(init)
    rc = lib.hgf_learn_host_run(T, ctypes.c_longlong(nb), iterations, P(pr), ctypes.c_float(z_precision),
                                ctypes.c_float(y_variance), P(ini), P(t), P(lw2), P(yy), P(out["x0"]), P(out["xz"]),
                                P(out["kw"]), P(out["hist_kw"]), P(out["free_energy"]), P(out["status"]))
    assert rc == 0
    return out


# Bounds of the fp32 kernel against the fp64 reference, per chain (the worst cases are recorded in DESIGN 3.19):
TOL_X = 1e-5      # q(x_0 .. x_T), q(z) means: relative L2 over t (TOL_MEAN)
TOL_XV = 1e-4     # their variances (TOL_COV)
TOL_KW_M = 5e-3   # q(kappa), q(omega) and their histories: mean error in units of the reference posterior's std
TOL_KW_V = 1e-4   # ... and variance error relative to the reference variance
FE_TOL = 1e-5     # relative to max(|F|, 1)
DEGENERATE = 1e-20  # a reference q(z_t) variance below this, in any update, may be flagged by the fp32 kernel (gate)


def per_chain_rel(got, want):
    ax = tuple(range(got.ndim - 1))
    return (np.sqrt(((got - want) ** 2).sum(ax)) / np.maximum(np.sqrt((want ** 2).sum(ax)), 1e-30)).max()


def kw_errors(got, want):
    """(mean error / reference std, variance error / reference variance) of [..., 2 (kappa, omega), 2 (m, v), batch]."""
    m, v = want[..., 0, :], want[..., 1, :]
    return (np.abs(got[..., 0, :] - m) / np.sqrt(v)).max(), (np.abs(got[..., 1, :] - v) / v).max()


def gate(case, r, ref):
    """Every chain against the reference at the bounds above; returns the worst error of each output.  q(x_0) is gated
    with q(x) as its first row.  A chain on which the reference itself breaks down (a GH product collapsing to a zero
    variance, then non-finite values) must be flagged.  A chain whose reference q(z_t) variance falls below DEGENERATE
    in any update (a GH product resolved by one node, beyond what fp32 holds) may be flagged; every other chain carries
    status 0.  The flagged chains are left out of the comparison."""
    g = lambda k: np.asarray(r[k], np.float64)
    nb = g("xz").shape[-1]
    bad = ~np.isfinite(ref["xz"].reshape(-1, nb)).all(0) | ~np.isfinite(ref["kw"].reshape(-1, nb)).all(0)
    with np.errstate(invalid="ignore"):
        degenerate = bad | ~(ref["min_vz"] >= DEGENERATE)
    status = np.asarray(r["status"])
    assert np.all(status[bad] != 0) and np.all(status[~degenerate] == 0), (case, status, bad, degenerate)
    ok = status == 0
    rows = lambda xz, x0, i: np.concatenate([x0[i:i + 1], xz[:, i], xz[:, i + 2]])[..., ok]
    errs = {"x_mean": per_chain_rel(rows(g("xz"), g("x0"), 0), rows(ref["xz"], ref["x0"], 0)),
            "x_var": per_chain_rel(rows(g("xz"), g("x0"), 1), rows(ref["xz"], ref["x0"], 1))}
    for k in ("kw", "hist_kw"):
        if r.get(k) is not None:
            errs[k + "_mean"], errs[k + "_var"] = kw_errors(g(k)[..., ok], ref[k][..., ok])
    if r.get("free_energy") is not None:
        fe, fr = g("free_energy")[..., ok], ref["free_energy"][..., ok]
        errs["free_energy"] = (np.abs(fe - fr) / np.maximum(np.abs(fr), 1.0)).max()
    tol = dict(x_mean=TOL_X, x_var=TOL_XV, kw_mean=TOL_KW_M, kw_var=TOL_KW_V, hist_kw_mean=TOL_KW_M, hist_kw_var=TOL_KW_V,
               free_energy=FE_TOL)
    for k, e in errs.items():
        assert e < tol[k], f"{case}: {k} {e:.3g} (bound {tol[k]:g})"
    return errs


def reference_on_f32(y, its, h):
    return hgf_learn(np.asarray(y, np.float32).astype(np.float64), its, **f32(h))


@pytest.mark.parametrize("hyper", sorted(HYPER))
def test_kernel_body_on_the_host_matches_the_reference(hyper):
    lib = _host_harness()
    h = HYPER[hyper]
    for T in (1, 2, 7, 300):
        for its in (1, 20):
            y = series(T, 3, seed=T + its, p_missing=0.2 if T > 2 else 0.0)
            r = run_host(lib, y, its, **h)
            gate(f"{hyper} T={T} its={its}", r, reference_on_f32(y, its, h))


def test_kernel_body_on_the_host_flags_bad_chains_only():
    """A chain with an infinite observation is flagged RXG_ERR_NAN; its neighbours keep their results."""
    lib = _host_harness()
    y = series(30, 4, seed=21, p_missing=0.1)
    y[12, 2] = np.inf
    r = run_host(lib, y, 4, **SET_B)
    assert list(r["status"]) == [0, 0, 5, 0]
    keep = [0, 1, 3]
    ref = reference_on_f32(y[:, keep], 4, SET_B)
    sub = {k: (v[..., keep] if isinstance(v, np.ndarray) else v) for k, v in r.items()}
    gate("neighbours of an inf chain", sub, ref)


def test_kernel_body_on_the_host_without_free_energy_computes_the_same():
    lib = _host_harness()
    y = series(25, 3, seed=4, p_missing=0.2)
    a = run_host(lib, y, 6, **SET_C)
    b = run_host(lib, y, 6, **SET_C, want_free_energy=False)
    for k in ("x0", "xz", "kw", "hist_kw", "status"):
        assert np.array_equal(a[k], b[k]), k


def test_kernel_body_on_the_host_reference_configuration():
    lib = _host_harness()
    y = reference_data()
    r = run_host(lib, y, 10, **DEFAULT)
    hgf1_assertions(r["xz"][:, 0], r["xz"][:, 1], r["free_energy"])
    gate("hgf_1", r, reference_on_f32(y, 10, DEFAULT))


# --------------------------------------------------------------------------- host-side argument handling
def test_infer_argument_handling(rx):
    """infer refuses everything outside the batched path before it needs a device (context=object() would fail on any
    use), so these run with and without a GPU."""
    from rxinfer_jl_b200 import BetheFactorization, KeepEach, KeepLast, MeanField, NormalMeanVariance, hgf_offline
    from rxinfer_jl_b200.inference import hgf_offline_arguments
    init = {"κ": NormalMeanVariance(0.9, 0.5), "ω": NormalMeanVariance(-0.1, 0.4), "z": NormalMeanVariance(0.2, 0.3),
            "x": NormalMeanVariance(0.1, 2.0)}
    model = hgf_offline(κ_prior=(0.7, 0.3), ω_prior=(-0.4, 0.5), x0_prior=(0.2, 2.0), z1_prior=(-0.3, 0.6), z_precision=2.5,
                        y_variance=0.3)
    args = hgf_offline_arguments(model, init)
    assert args["prior"] == list(SET_B["prior"]) and args["z_precision"] == 2.5 and args["y_variance"] == 0.3
    assert args["init"] == [0.9, 0.5, -0.1, 0.4, 0.2, 0.3, 0.1, 2.0]
    assert hgf_offline_arguments(hgf_offline(), {k: NormalMeanVariance(*v) for k, v in
                                                 zip(("κ", "ω", "z", "x"), ((1.0, 1.0), (0.0, 1.0), (0.0, 1.0), (0.0, 1.0)))}) == \
        dict(prior=list(DEFAULT["prior"]), init=list(DEFAULT["init"]), z_precision=1.0, y_variance=1.0)
    y = np.zeros((5, 2), np.float32)
    call = lambda **kw: rx.infer(**{**dict(model=model, data={"y": y}, constraints=MeanField(), initialization=init,
                                            iterations=3, context=object()), **kw})
    for c in (None, BetheFactorization(), "q(x)q(z)"):
        with pytest.raises(ValueError, match="mean-field"):
            call(constraints=c)
    with pytest.raises(ValueError, match="initialization"):
        call(initialization={k: v for k, v in init.items() if k != "ω"})
    with pytest.raises(ValueError, match="initialization"):
        call(initialization=None)
    with pytest.raises(NotImplementedError, match="predictvars"):
        call(predictvars={"y": KeepLast()})
    with pytest.raises(ValueError, match="mutually exclusive"):
        call(datastream=iter([y]))
    with pytest.raises(NotImplementedError, match="datastream"):
        call(data=None, datastream=iter([y]))
    with pytest.raises(KeyError, match="y"):
        call(data={"x": y})
    for rv in (KeepEach(), {"x": KeepEach()}, {"z": KeepEach()}, {"θ": KeepLast()}):
        with pytest.raises(NotImplementedError, match="returnvars"):
            call(returnvars=rv)


def test_julia_shim_reads_kappa_and_omega_by_variable():
    """The shim downloads the ABI's kw[2 (κ, ω)][2 (m, v)][batch] column-major as kw[b, (m, v), (κ, ω)]: q(κ) is
    (kw[b, 1, 1], kw[b, 2, 1]) and q(ω) is (kw[b, 1, 2], kw[b, 2, 2]).  Julia cannot run here, so the index pattern is
    checked in the source."""
    jl = open(os.path.join(ROOT, "rxinfer.jl_b200", "julia", "RxGaussB200.jl")).read()
    assert ":κ => [NormalMeanVariance(Float64(kw[b, 1, 1]), Float64(kw[b, 2, 1])) for b in 1:batch]" in jl
    assert ":ω => [NormalMeanVariance(Float64(kw[b, 1, 2]), Float64(kw[b, 2, 2])) for b in 1:batch]" in jl
