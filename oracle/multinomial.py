"""fp64 restatement of mean-field Pólya-Gamma VMP for Bayesian multinomial regression (MultinomialPolya node; DESIGN 3.22).

    ψ ~ MvNormalWeightedMeanPrecision(ξ0, W0);  y[i] ~ MultinomialPolya(N_i, ψ),  y_i ∈ ℕ^K,  D = K − 1

read through stick-breaking: y_ik ~ Binomial(N_ik, σ(ψ_k)), k = 1..D, N_ik = N_i − Σ_{j<k} y_ij.  Written from the message
form and deliberately not collapsed: every sample sends ψ its own message MvNormalWeightedMeanPrecision(b_i,
diag(N_ik E[ω_ik])) with b_ik = y_ik − N_ik/2 and E[ω] the Pólya-Gamma mean at c_k = sqrt(m_k² + Σ_kk) under q(ψ); q(ψ) is
the product of the base and the messages, by dense inverses; the free energy is summed sample by sample.  A sample with a
negative count is read as all-zero and flags its chain.  Arrays of one chain: y [n, K]."""
import numpy as np
from scipy.special import expit, gammaln

from oracle.binomial import LOG2, kl_gauss, log_cosh_half, omega_bar


def stick_breaking(psi):
    """p = logistic_stick_breaking(ψ): p_1 = σ(ψ_1), p_k = σ(ψ_k)(1 − Σ_{j<k} p_j), p_K = 1 − Σ_{j<K} p_j."""
    psi = np.asarray(psi, np.float64)
    p = np.empty(len(psi) + 1)
    rest = 1.0
    for k, s in enumerate(expit(psi)):
        p[k] = s * rest
        rest -= p[k]
    p[-1] = rest
    return p


def binomials(y):
    """The stick-breaking binomials of samples y [n, K]: trials N_ik and successes y_ik, [n, D] each."""
    y = np.asarray(y, np.float64)
    N = np.cumsum(y[:, ::-1], axis=1)[:, ::-1]          # N_ik = Σ_{j >= k} y_ij
    return N[:, :-1], y[:, :-1]


def log_coefficient(y):
    """log multinomial coefficient of every sample, [n]."""
    y = np.asarray(y, np.float64)
    return gammaln(y.sum(1) + 1) - gammaln(y + 1).sum(1)


def valid(y):
    return (np.asarray(y) >= 0).all(axis=1)


def messages(y, m, S):
    """Per sample: b_i [n, D] and the diagonal precision [n, D] of its message to ψ at q(ψ) = N(m, S)."""
    Nk, yk = binomials(y)
    c = np.sqrt(m ** 2 + np.diag(S))
    return yk - Nk / 2, omega_bar(Nk, c[None, :])


def free_energy(y, m0, S0, m, S):
    """F(q) = KL(q ‖ base) − Σ_i [log C_i − Σ_k N_ik log 2 + Σ_k b_ik m_k − Σ_k N_ik log cosh(c_k/2)], c at q; the base
    N(m0, S0) in moment form."""
    Nk, yk = binomials(y)
    c = np.sqrt(m ** 2 + np.diag(S))
    b = yk - Nk / 2
    per = log_coefficient(y) - LOG2 * Nk.sum(1) + b @ m - (Nk * log_cosh_half(c)[None]).sum(1)
    return kl_gauss(m, S, np.linalg.solve(S0, m0), np.linalg.inv(S0)) - per.sum()


def free_energy_uncollapsed(y, m0, S0, m, S, cq):
    """F of q(ψ) q(ω) with q(ω_ik) = PG(N_ik, cq_k): KL(q(ψ)) + Σ KL(PG(N, cq) ‖ PG(N, 0)) − E[log p(y | ψ, ω)]."""
    Nk, yk = binomials(y)
    e2 = m ** 2 + np.diag(S)
    w = omega_bar(Nk, cq[None, :])
    kl_w = Nk * log_cosh_half(cq)[None] - cq[None] ** 2 * w / 2
    b = yk - Nk / 2
    ll = log_coefficient(y) - LOG2 * Nk.sum(1) + b @ m - (w * e2[None]).sum(1) / 2
    return kl_gauss(m, S, np.linalg.solve(S0, m0), np.linalg.inv(S0)) + kl_w.sum() - ll.sum()


def step(y, m0, S0, m, S):
    """q = base N(m0, S0) ⊗ every sample's message at the current q = N(m, S), by dense inverses."""
    b, w = messages(y, m, S)
    W0 = np.linalg.inv(S0)
    Lam = W0 + np.diag(w.sum(0))
    Sn = np.linalg.inv(Lam)
    Sn = (Sn + Sn.T) / 2
    return Sn @ (W0 @ m0 + b.sum(0)), Sn


def collapsed_step(b, n, m0, S0, m, S):
    """The kernels' step on a message (b, n): d = n g(c), D Sherman–Morrison updates of S0, m = m0 + Σ(b − d∘m0), and
    KL(q ‖ base) from the byproducts: ½[(m − m0)ᵀ(b − d∘m) − Σ d_k Σ_kk + Σ log pivot_k].  Returns m, Σ, KL."""
    d = omega_bar(n, np.sqrt(m ** 2 + np.diag(S)))
    Sn = np.array(S0, np.float64)
    logdet = 0.0
    for k in range(len(d)):
        if d[k] == 0:
            continue
        u = Sn[k].copy()
        piv = 1 + d[k] * u[k]
        Sn -= d[k] / piv * np.outer(u, u)
        logdet += np.log(piv)
    mn = m0 + Sn @ (b - d * m0)
    return mn, Sn, 0.5 * ((mn - m0) @ (b - d * mn) - d @ np.diag(Sn) + logdet)


def vmp(y, xi0, W0, iterations):
    """Whole data set, one chain: q_{k+1} = prior ⊗ the messages at q_k, from the prior.  Returns means [its, D],
    covariances [its, D, D], free energies [its] and whether a sample was unusable."""
    y = np.asarray(y, np.float64)
    ok = valid(y)
    y = np.where(ok[:, None], y, 0.0)
    S0 = np.linalg.inv(np.asarray(W0, np.float64))
    m0 = S0 @ np.asarray(xi0, np.float64)
    m, S = m0, S0
    means, covs, fes = [], [], []
    for _ in range(iterations):
        m, S = step(y, m0, S0, m, S)
        means.append(m)
        covs.append(S)
        fes.append(free_energy(y, m0, S0, m, S))
    return dict(mean=np.array(means), cov=np.array(covs), free_energy=np.array(fes), bad=not bool(ok.all()))


def online(y, xi0, W0, iterations=1, m=None, S=None):
    """Datum by datum, one chain: datum t runs `iterations` steps from the base q_{t−1}; q_0 = N(W0⁻¹ξ0, W0⁻¹) unless a
    carry (m, S) is given.  Returns per datum means [T, D], covariances [T, D, D], free energies [T] (KL(q_t ‖ q_{t−1})
    minus datum t's bound), the final (m, S) and whether a datum was unusable."""
    y = np.asarray(y, np.float64)
    ok = valid(y)
    y = np.where(ok[:, None], y, 0.0)
    if m is None:
        S = np.linalg.inv(np.asarray(W0, np.float64))
        m = S @ np.asarray(xi0, np.float64)
    means, covs, fes = [], [], []
    for t in range(len(y)):
        m0, S0 = m, S
        for _ in range(iterations):
            m, S = step(y[t:t + 1], m0, S0, m, S)
        means.append(m)
        covs.append(S)
        fes.append(free_energy(y[t:t + 1], m0, S0, m, S))
    return dict(mean=np.array(means), cov=np.array(covs), free_energy=np.array(fes), m=m, S=S, bad=not bool(ok.all()))


def _stack(outs, keys):
    return {k: np.stack([o[k] for o in outs], -1) for k in keys}


def vmp_batch(y, xi0, W0, iterations):
    """``vmp`` of every chain in the kernel's layout y [n, K, batch]: hist_mean [its, D, batch], hist_cov
    [its, D, D, batch], free_energy [its, batch], bad [batch]."""
    outs = [vmp(y[:, :, b], xi0, W0, iterations) for b in range(y.shape[2])]
    r = _stack(outs, ("mean", "cov", "free_energy", "bad"))
    return dict(hist_mean=r["mean"], hist_cov=r["cov"], free_energy=r["free_energy"], bad=r["bad"])


def online_batch(y, xi0, W0, iterations=1):
    """``online`` of every chain in the kernel's layout y [T, K, batch]: hist_mean [T, D, batch], hist_cov [T, D, D, batch],
    free_energy [T, batch], m [D, batch], S [D, D, batch], bad [batch]."""
    outs = [online(y[:, :, b], xi0, W0, iterations) for b in range(y.shape[2])]
    r = _stack(outs, ("mean", "cov", "free_energy", "m", "S", "bad"))
    return dict(hist_mean=r["mean"], hist_cov=r["cov"], free_energy=r["free_energy"], m=r["m"], S=r["S"], bad=r["bad"])
