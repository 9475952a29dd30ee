"""The fp64 oracles of the five small VMP models, checked at non-default hyper-parameters against computations that do
not share their code: the GCV rules against scipy.integrate.quad of the defining densities, the AR regression VMP
against the conjugate updates from the dense design matrix, the IID Wishart VMP against the updates from the sufficient
statistics, and the free energies of the Gamma models against their definitions.  The reference's own tests pin these
oracles only at kappa = 1, omega = 0 and unit priors; tests/test_vmp_models_gpu.py relies on them elsewhere."""
import numpy as np
import pytest
from scipy import integrate, stats
from scipy.special import digamma, gammaln, roots_legendre

from oracle import hgf, vmp
from oracle import rules as R

KAPPA_OMEGA = [(0.6, -0.8), (1.7, 0.5)]


def _quad(f, lo, hi):
    return integrate.quad(f, lo, hi, epsabs=0.0, epsrel=1e-12, limit=200)[0]


@pytest.mark.parametrize("kappa,omega", KAPPA_OMEGA)
def test_gcv_marginal_yx_against_quadrature(kappa, omega):
    """q(y, x) ∝ N(y; m_y, v_y) N(x; m_x, v_x) exp(E_q(z)[log N(y; x, exp(kappa z + omega))]): the (y, x)-dependent part
    of the expectation is -(y - x)^2 E[exp(-kappa z - omega)] / 2, with E taken by quad over q(z).  The moments of the
    smooth, Gaussian-tailed 2-D density come from a 300 x 300 Gauss-Legendre product rule over +-12 prior sd (converged
    far below the bounds; adaptive 2-D quad takes minutes here)."""
    t, wl = roots_legendre(300)
    for (my, vy), (mx, vx), (mz, vz) in (((0.4, 0.05), (-0.3, 0.8), (0.2, 0.3)), ((-1.2, 0.3), (0.5, 0.2), (-0.6, 0.9))):
        sz = np.sqrt(vz)
        g = _quad(lambda z: stats.norm.pdf(z, mz, sz) * np.exp(-kappa * z - omega), mz - 40 * sz, mz + 40 * sz)
        hy, hx = 12 * np.sqrt(vy), 12 * np.sqrt(vx)
        Y, X = np.meshgrid(my + hy * t, mx + hx * t, indexing="ij")
        W = np.outer(wl, wl) * stats.norm.pdf(Y, my, np.sqrt(vy)) * stats.norm.pdf(X, mx, np.sqrt(vx)) * np.exp(-0.5 * g * (Y - X) ** 2)
        W /= W.sum()
        Ey, Ex = (W * Y).sum(), (W * X).sum()
        Vyy, Vxx, Vyx = (W * (Y - Ey) ** 2).sum(), (W * (X - Ex) ** 2).sum(), (W * (Y - Ey) * (X - Ex)).sum()
        m, V = R.gcv_marginal_yx((np.array([my]), np.array([vy])), (np.array([mx]), np.array([vx])),
                                 (np.array([mz]), np.array([vz])), kappa, omega)
        assert abs(R.gcv_gamma((mz, vz), kappa, omega) - g) < 1e-12 * g
        assert np.allclose(m[0], [Ey, Ex], rtol=0, atol=1e-9), (m[0], Ey, Ex)
        assert np.allclose(V[0], [[Vyy, Vyx], [Vyx, Vxx]], rtol=1e-8, atol=1e-11), (V[0], Vyy, Vyx, Vxx)


# (prior mean, prior variance, psi) of the z product: the range the filter runs in (q(z) variances up to ~0.5, psi up to a
# few); GH-31 meets GH31_TOL there, a GH-101 rule agrees with the quadrature to GH101_TOL (it checks the quadrature)
Z_CASES = [(0.3, 0.5, 0.8), (0.1, 0.05, 0.2), (-0.4, 0.3, 1.5), (0.8, 0.2, 4.0)]
GH31_TOL = (2e-6, 1e-5)                 # |mean error|, relative variance error
GH101_TOL = (1e-10, 1e-9)


@pytest.mark.parametrize("kappa,omega", KAPPA_OMEGA)
def test_gcv_z_product_against_quadrature(kappa, omega):
    """q(z) ∝ N(z; mu0, v0) exp(-(kappa z + omega) / 2 - psi exp(-kappa z - omega) / 2): the product of the prior with the
    ExponentialLinearQuadratic message of rules.gcv_z_elq, moments by rules.prod_normal_elq (GH-31) against quad."""
    for mu0, v0, psi in Z_CASES:
        f = lambda z: np.exp(-0.5 * (z - mu0) ** 2 / v0 - 0.5 * (kappa * z + omega) - 0.5 * psi * np.exp(-kappa * z - omega))
        lo, hi = mu0 - 40 * np.sqrt(v0), mu0 + 40 * np.sqrt(v0)
        Z = _quad(f, lo, hi)
        mq = _quad(lambda z: z * f(z), lo, hi) / Z
        vq = _quad(lambda z: (z - mq) ** 2 * f(z), lo, hi) / Z
        # the joint q(y, x) enters only through psi = E(y - x)^2
        m = np.array([[0.5, 0.5 - np.sqrt(psi / 2)]])
        V = np.array([[[psi / 3, psi / 12], [psi / 12, psi / 3]]])          # psi/2 + psi/3 + psi/3 - psi/6 = psi
        elq = R.gcv_z_elq(m, V, kappa, omega)
        assert abs(elq[1][0] - psi * np.exp(-omega)) < 1e-12 * psi
        prior = (np.array([mu0]), np.array([v0]))
        for nw, (tm, tv) in ((None, GH31_TOL), (R.gauss_hermite(101), GH101_TOL)):
            mz, vz = R.prod_normal_elq(prior, elq, nw)
            assert abs(mz[0] - mq) < tm and abs(vz[0] - vq) < tv * vq, (mu0, v0, psi, mz[0] - mq, vz[0] / vq - 1)


@pytest.mark.parametrize("kappa,omega", KAPPA_OMEGA)
def test_hgf_free_energy_non_increasing(kappa, omega):
    """The reference's assertion for this model (free energy averaged over the data, per iteration, does not increase),
    at kappa != 1, omega != 0."""
    zv, yv = (0.0625, 0.015625) if kappa < 1 else (0.015625, 0.03125)
    _, _, y = hgf.generate_data(200, 16, kappa=kappa, omega=omega, z_variance=zv, y_variance=yv, seed=3)
    _, fe = hgf.hgf_filter(y, iters=10, kappa=kappa, omega=omega, z_variance=zv, y_variance=yv, init=(0.3, 2.5, -0.4, 3.0),
                           return_free_energy=True)
    hist = fe.mean(axis=0)                                          # [iterations, chain]
    assert np.all(np.diff(hist, axis=0) <= 1e-6 * np.abs(hist[:-1]))
    assert np.all(hist[-1] < hist[0])


def _lags(s, p):
    """Dense design matrix of the AR regression for one series: row k = (s[k+p-1], ..., s[k]), target s[k+p]."""
    n = len(s) - p
    X = np.empty((n, p))
    for k in range(n):
        for j in range(p):
            X[k, j] = s[k + p - 1 - j]
    return X, s[p:]


def test_ar_regression_against_dense_conjugate_updates():
    """Order 8, non-unit priors: q(theta) = N(V E[g] X'y, V = (w0 I + E[g] X'X)^-1), q(g) = Gamma(a0 + n/2,
    b0 + (|y - X m|^2 + tr(X'X V)) / 2), and the free energy E_q[log q - log p] from scipy's densities and entropies."""
    rng = np.random.default_rng(5)
    p, N, its = 8, 60, 6
    a0, b0, w0, ia, ib = 2.5, 0.5, 0.3, 3.0, 2.0
    s = np.zeros((N, 3))
    s[:, 0] = rng.standard_normal(N)
    for k in range(2, N):
        s[k, 1] = 0.5 * s[k - 1, 1] - 0.3 * s[k - 2, 1] + 0.7 * rng.standard_normal()
    s[:, 2] = np.cumsum(rng.standard_normal(N)) * 0.2 + 1.0
    r = vmp.ar_regression(s, p, iterations=its, gamma_prior=(a0, b0), theta_prior_precision=w0, init_gamma=(ia, ib))
    for c in range(3):
        X, y = _lags(s[:, c], p)
        n = len(y)
        ga, gb = ia, ib
        for it in range(its):
            Eg = ga / gb
            V = np.linalg.inv(w0 * np.eye(p) + Eg * X.T @ X)
            m = V @ (Eg * X.T @ y)
            ga, gb = a0 + n / 2, b0 + 0.5 * (np.sum((y - X @ m) ** 2) + np.trace(X.T @ X @ V))
            Elog, Eg = digamma(ga) - np.log(gb), ga / gb
            E_lik = -0.5 * n * np.log(2 * np.pi) + 0.5 * n * Elog - 0.5 * Eg * (np.sum((y - X @ m) ** 2) + np.trace(X.T @ X @ V))
            E_th = -0.5 * p * np.log(2 * np.pi) + 0.5 * p * np.log(w0) - 0.5 * w0 * (np.trace(V) + m @ m)
            E_g = a0 * np.log(b0) - gammaln(a0) + (a0 - 1) * Elog - b0 * Eg
            H = stats.multivariate_normal(m, V).entropy() + stats.gamma(ga, scale=1.0 / gb).entropy()
            assert abs(r["free_energy"][it, c] - (-E_lik - E_th - E_g - H)) < 1e-9 * abs(r["free_energy"][it, c]), (c, it)
        assert np.allclose(r["theta_mean"][:, c], m, rtol=1e-10, atol=1e-12)
        assert np.allclose(r["theta_cov"][:, :, c], V, rtol=1e-10, atol=1e-14)
        assert abs(r["gamma_shape"][c] - ga) < 1e-12 and abs(r["gamma_rate"][c] - gb) < 1e-10 * gb


def test_mv_iid_wishart_against_sufficient_statistic_updates():
    """Non-zero mu0, non-identity inv_scale0 and Lambda0, nu0 != d + 1: per iteration Lambda = Lambda0 + N E[P],
    m = Lambda^-1 (Lambda0 mu0 + E[P] sum y), inv_scale = inv_scale0 + sum y y' - sum y m' - m sum y' + N (m m' + V),
    E[P] = (nu0 + N) inv(inv_scale) -- the update the CUDA kernel implements."""
    rng = np.random.default_rng(9)
    d, N, batch, its = 3, 25, 4, 5
    mu0 = np.array([0.8, -0.5, 1.2])
    M = rng.standard_normal((d, d))
    L0, iS0 = M @ M.T + 0.5 * np.eye(d), np.array([[2.0, 0.4, -0.2], [0.4, 1.5, 0.3], [-0.2, 0.3, 0.8]])
    nu0 = d + 2.5
    EP0 = np.array([[1.2, 0.3, 0.0], [0.3, 0.9, -0.2], [0.0, -0.2, 1.1]])
    y = rng.standard_normal((N, d, batch)) + rng.standard_normal((1, d, batch))
    r = vmp.mv_iid_wishart(y, iterations=its, mu0=mu0, Lambda0=L0, nu0=nu0, inv_scale0=iS0, init_E_P=EP0)
    for b in range(batch):
        sy, syy = y[:, :, b].sum(0), y[:, :, b].T @ y[:, :, b]
        EP = EP0
        for _ in range(its):
            V = np.linalg.inv(L0 + N * EP)
            m = V @ (L0 @ mu0 + EP @ sy)
            iS = iS0 + syy - np.outer(sy, m) - np.outer(m, sy) + N * (np.outer(m, m) + V)
            EP = (nu0 + N) * np.linalg.inv(iS)
        assert np.allclose(r["m_mean"][:, b], m, rtol=1e-11, atol=1e-13)
        assert np.allclose(r["m_cov"][:, :, b], V, rtol=1e-11, atol=1e-15)
        assert np.allclose(r["inv_scale"][:, :, b], iS, rtol=1e-11, atol=1e-12)
        assert r["df"][b] == nu0 + N


@pytest.mark.parametrize("a", [-0.9, 0.7])
def test_lgssm_gamma_free_energy_closed_form_equals_definition(a):
    """At A_scalar != 1 and non-default priors the closed form the CUDA kernel evaluates equals the dense evaluation of
    the definition, and it does not increase."""
    rng = np.random.default_rng(3)
    T, batch = 25, 4
    x = np.zeros((T, batch))
    for t in range(1, T):
        x[t] = a * x[t - 1] + np.sqrt(0.6) * rng.standard_normal(batch)
    y = x + rng.standard_normal((T, batch)) / np.sqrt(rng.gamma(2.0, 1.0, batch) + 0.3)
    r = vmp.lgssm_gamma_precision(y, A_scalar=a, prior=(1.5, 2.0), proc_var=0.6, gamma_prior=(2.0, 3.0), iterations=6,
                                  init_Etau=0.4, return_free_energy=True)
    assert np.allclose(r["free_energy"], r["free_energy_closed_form"], rtol=0, atol=1e-8)
    assert np.all(np.diff(r["free_energy"], axis=0) < 1e-10)


@pytest.mark.parametrize("w", [0.3, 3.0])
def test_stream_vmp_gamma_free_energy_non_increasing(w):
    """Per datum, the mean-field free energy does not increase over the iterations at w != 1 with a non-default
    initialisation (every update is a coordinate minimisation of it)."""
    rng = np.random.default_rng(1)
    x = np.cumsum(rng.standard_normal((50, 32)) / np.sqrt(w), axis=0)
    y = x + rng.standard_normal((50, 32)) / np.sqrt(rng.gamma(2.0, 1.0, 32) + 0.2)
    _, fe = vmp.stream_vmp_gamma(y, iterations=5, w=w, init_x=(0.5, 20.0), init_tau=(2.0, 1.5), return_free_energy=True)
    assert np.all(np.diff(fe, axis=1) <= 1e-12 * np.abs(fe[:, :-1]))
