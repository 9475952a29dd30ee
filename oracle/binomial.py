"""fp64 restatement of mean-field Pólya-Gamma VMP for Bayesian binomial regression (BinomialPolya node; DESIGN 3.21).

    β ~ MvNormalWeightedMeanPrecision(ξ0, W0);  y[i] ~ BinomialPolya(x[i], n[i], β)  (y_i ~ Binomial(n_i, σ(x_iᵀβ)))

Written from the message form: each node sends β the message MvNormalWeightedMeanPrecision((y_i − n_i/2) x_i,
E[ω_i] x_i x_iᵀ) with E[ω_i] the Pólya-Gamma mean at c_i = sqrt(E[(x_iᵀβ)²]) under q(β), and q(β) is the product of the
prior and the N messages.  The free energy of a Gaussian q is the collapsed Pólya-Gamma (Jaakkola–Jordan) bound.  A
sample with n = 0 sends the uniform message.  Arrays of one chain: X [N, p], y [N], n [N]."""
import numpy as np
from scipy.special import gammaln

LOG2 = np.log(2.0)


def omega_bar(n, c):
    """E[ω] of PG(n, c) = n tanh(c/2) / (2c), n/4 − n c²/48 near c = 0."""
    c = np.abs(np.asarray(c, np.float64))
    small = c < 1e-4
    cs = np.where(small, 1.0, c)
    return np.asarray(n, np.float64) * np.where(small, 0.25 - c * c / 48.0, np.tanh(cs / 2) / (2 * cs))


def log_cosh_half(c):
    """log cosh(c/2) in its stable form |c|/2 + log1p(e^−|c|) − log 2."""
    c = np.abs(np.asarray(c, np.float64))
    return c / 2 + np.log1p(np.exp(-c)) - LOG2


def message(x, y, n, m, S):
    """The BinomialPolya node's message to β at q(β) = N(m, S), weighted-mean / precision form; c at q as well."""
    psi = x @ m
    c = np.sqrt(psi ** 2 + np.einsum("ij,jk,ik->i", x, S, x))
    w = omega_bar(n, c)
    return (y - n / 2)[:, None] * x, w[:, None, None] * x[:, :, None] * x[:, None, :], c


def kl_gauss(m, S, xi0, W0):
    """KL(N(m, S) || N(W0⁻¹ ξ0, W0⁻¹))."""
    p = len(m)
    d = m - np.linalg.solve(W0, xi0)
    return 0.5 * (np.trace(W0 @ S) + d @ W0 @ d - p - np.linalg.slogdet(S)[1] - np.linalg.slogdet(W0)[1])


def free_energy(X, y, n, xi0, W0, m, S):
    """The collapsed bound F(q) = KL(q ‖ prior) − Σ [log C(n, y) − n log 2 + (y − n/2) ψ − n log cosh(c/2)]."""
    psi = X @ m
    c = np.sqrt(psi ** 2 + np.einsum("ij,jk,ik->i", X, S, X))
    lc = gammaln(n + 1.0) - gammaln(y + 1.0) - gammaln(n - y + 1.0)
    return kl_gauss(m, S, xi0, W0) - np.sum(lc - n * LOG2 + (y - n / 2) * psi - n * log_cosh_half(c))


def free_energy_uncollapsed(X, y, n, xi0, W0, m, S, cq):
    """F of q(β) q(ω) with q(ω_i) = PG(n_i, cq_i): KL(q(β)) + Σ KL(PG(n, cq) ‖ PG(n, 0)) − E[log p(y | β, ω)], where
    p(y | ψ, ω) = C(n, y) 2^−n exp((y − n/2) ψ − ω ψ²/2) and KL(PG(n, c') ‖ PG(n, 0)) = n log cosh(c'/2) − c'² E[ω]/2."""
    psi = X @ m
    e2 = psi ** 2 + np.einsum("ij,jk,ik->i", X, S, X)
    w = omega_bar(n, cq)
    lc = gammaln(n + 1.0) - gammaln(y + 1.0) - gammaln(n - y + 1.0)
    kl_w = n * log_cosh_half(cq) - np.asarray(cq, np.float64) ** 2 * w / 2
    return kl_gauss(m, S, xi0, W0) + np.sum(kl_w) - np.sum(lc - n * LOG2 + (y - n / 2) * psi - w * e2 / 2)


def valid_samples(X, y, n):
    """Per sample: usable (finite x, 0 <= y <= n); an unusable one is read as n = 0 and flags its chain."""
    return np.isfinite(X).all(axis=1) & (y >= 0) & (n >= y)


def vmp(X, y, n, xi0, W0, iterations, want_free_energy=True):
    """Mean-field VMP of one chain from the prior: per iteration the product of the prior and the N messages at the
    previous q.  Returns the per-iteration means [its, p], covariances [its, p, p], free energies [its] (of the posterior
    each iteration returns) and whether a sample was unusable."""
    X = np.asarray(X, np.float64)
    y = np.asarray(y, np.float64)
    n = np.ones(len(y)) if n is None else np.asarray(n, np.float64)
    xi0 = np.asarray(xi0, np.float64)
    W0 = np.asarray(W0, np.float64)
    ok = valid_samples(X, y, n)
    X, y, n = np.where(ok[:, None], X, 0.0), np.where(ok, y, 0.0), np.where(ok, n, 0.0)
    S = np.linalg.inv(W0)
    m = S @ xi0
    means, covs, fes = [], [], []
    for _ in range(iterations):
        xi_msg, W_msg, _ = message(X, y, n, m, S)
        xi, W = xi0 + xi_msg.sum(0), W0 + W_msg.sum(0)
        S = np.linalg.inv(W)
        S = (S + S.T) / 2
        m = S @ xi
        means.append(m)
        covs.append(S)
        if want_free_energy:
            fes.append(free_energy(X, y, n, xi0, W0, m, S))
    return dict(mean=np.array(means), cov=np.array(covs), free_energy=np.array(fes) if want_free_energy else None,
                bad=not bool(ok.all()))


def vmp_batch(X, y, n, xi0, W0, iterations, want_free_energy=True):
    """``vmp`` of every chain in the kernel's layout: X [N, p, batch], y and n [N, batch] (n None: Bernoulli).  Returns
    hist_mean [its, p, batch], hist_cov [its, p, p, batch], free_energy [its, batch], bad [batch]."""
    outs = [vmp(X[:, :, b], y[:, b], None if n is None else n[:, b], xi0, W0, iterations, want_free_energy)
            for b in range(X.shape[2])]
    return dict(hist_mean=np.stack([o["mean"] for o in outs], -1), hist_cov=np.stack([o["cov"] for o in outs], -1),
                free_energy=np.stack([o["free_energy"] for o in outs], -1) if want_free_energy else None,
                bad=np.array([o["bad"] for o in outs]))
