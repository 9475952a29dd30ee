"""Gaussian mixture VMP (rxg_gmm_vmp_f32) on the CPU: an fp64 reference written message by message, checked against
independent computations -- the closed-form free energy against its dense definition (scipy entropies), every update
against the conjugate sufficient-statistic update, a non-increasing free energy, the Beta / Gamma spelling against a
scalar VMP written with Beta and Gamma, the assertions of the reference's two mixture tests on data drawn from the same
models, and the argument handling of Context / infer."""
import numpy as np
import pytest
from scipy import stats
from scipy.special import digamma, gammaln, logsumexp, multigammaln

LOG2PI = np.log(2 * np.pi)
SCHEDULES = ("z_m_w_s", "z_w_m_s", "jacobi")


def _elogdet_w(nu, iS):
    """E[log|W|] of Wishart(nu, inv(iS)), nu[...], iS[..., d, d]."""
    d = iS.shape[-1]
    return sum(digamma(0.5 * (nu - i)) for i in range(d)) + d * np.log(2.0) - np.linalg.slogdet(iS)[1]


def gaussian_mixture(y, alpha0, mu0, V0, nu0, S0, alpha_init, m_init, Vm_init, nu_init, S_init, iterations=10,
                     schedule="z_m_w_s"):
    """Mean-field VMP of the Gaussian mixture (RxInfer test/models/mixtures/gmm_multivariate_tests.jl:4-24,
    constraints :76-80, initialization :26-64; gmm_univariate_tests.jl:6-26 is the d = 1, K = 2 case), fp64, batched over
    chains.  y[N, d, batch]; priors and initial marginals as in rxg_gmm_vmp_f32 (S0, S_init are Wishart scales).

    Messages, per point i and component k, with the current marginals (NormalMixture node, ReactiveMP's mean-field rules):
        to z[i]:   log rho_ik = E[log s_k] + 1/2 E[log|W_k|] - d/2 log 2 pi - 1/2 ((y_i - m_k)' E[W_k] (y_i - m_k) + tr(E[W_k] V_k))
                   (the Categorical node adds E[log s_k]); q(z_i) = softmax_k log rho_ik
        to m[k]:   MvNormal with precision r_ik E[W_k] and weighted mean r_ik E[W_k] y_i; q(m_k) = prior x prod_i
        to W[k]:   Wishart(1 + r_ik, inv(r_ik ((y_i - m_k)(y_i - m_k)' + V_k))) in the (df + d + 1, inverse scale) sense:
                   q(W_k) = Wishart(nu0 + sum_i r_ik, inv(inv(S0) + sum_i r_ik ((y_i - m_k)(y_i - m_k)' + V_k)))
        to s:      Dirichlet(1 + r_i); q(s) = Dirichlet(alpha0 + sum_i r_i)
    ``schedule`` orders one iteration: "z_m_w_s" (q(z); q(m) with the previous q(W); q(W) with the new q(m); q(s)),
    "z_w_m_s" (q(W) before q(m)) or "jacobi" (q(m), q(W) both from the previous iteration).  The free energy after every
    iteration is evaluated at the marginals then current, in closed form (``free_energy``)."""
    y = np.asarray(y, np.float64)
    N, d, B = y.shape
    Y = np.moveaxis(y, 2, 0)                                           # [B, N, d]
    K = len(alpha0)
    inv = np.linalg.inv
    alpha = np.tile(np.asarray(alpha_init, np.float64), (B, 1))
    m = np.tile(np.asarray(m_init, np.float64), (B, 1, 1))
    Vm = np.tile(np.asarray(Vm_init, np.float64), (B, 1, 1, 1))
    nu = np.tile(np.asarray(nu_init, np.float64), (B, 1))
    iS = np.tile(inv(np.asarray(S_init, np.float64)), (B, 1, 1, 1))
    V0i = inv(np.asarray(V0, np.float64)); S0i = inv(np.asarray(S0, np.float64))
    mu0 = np.asarray(mu0, np.float64); nu0 = np.asarray(nu0, np.float64)
    hist = {k: [] for k in ("alpha", "m_mean", "m_cov", "w_df", "w_inv_scale", "free_energy")}
    for _ in range(iterations):
        # ---- q(z)
        EW = nu[..., None, None] * inv(iS)
        lrho = log_rho(Y, alpha, m, Vm, nu, iS)
        r = np.exp(lrho - logsumexp(lrho, axis=2, keepdims=True))      # [B, N, K]
        Nk = r.sum(1)

        def update_m(EW_):
            # prior x the product of the per-point messages (r_ik E[W_k], r_ik E[W_k] y_i)
            W = V0i[None] + np.einsum("bnk,bkij->bkij", r, EW_)
            xi = np.einsum("kij,kj->ki", V0i, mu0)[None] + np.einsum("bnk,bkij,bnj->bki", r, EW_, Y)
            Vn = inv(W)
            return np.einsum("bkij,bkj->bki", Vn, xi), Vn

        def update_w(m_, Vm_):
            dy = Y[:, :, None, :] - m_[:, None]                           # [B, N, K, d]
            R = np.einsum("bnk,bnki,bnkj->bkij", r, dy, dy)
            return nu0[None] + Nk, S0i[None] + R + Nk[..., None, None] * Vm_

        if schedule == "z_m_w_s":
            m, Vm = update_m(EW)
            nu, iS = update_w(m, Vm)
        elif schedule == "z_w_m_s":
            nu, iS = update_w(m, Vm)
            m, Vm = update_m(nu[..., None, None] * inv(iS))
        elif schedule == "jacobi":
            m_n, Vm_n = update_m(EW)
            nu, iS = update_w(m, Vm)
            m, Vm = m_n, Vm_n
        else:
            raise ValueError(schedule)
        alpha = np.asarray(alpha0, np.float64)[None] + Nk
        fe = free_energy(Y, r, alpha, m, Vm, nu, iS, alpha0, mu0, V0, nu0, S0)
        for k, v in (("alpha", alpha.T), ("m_mean", np.moveaxis(m, 0, -1)), ("m_cov", np.moveaxis(Vm, 0, -1)),
                     ("w_df", nu.T), ("w_inv_scale", np.moveaxis(iS, 0, -1)), ("free_energy", fe)):
            hist[k].append(np.array(v))
    out = {"hist_" + k: np.stack(v) for k, v in hist.items() if k != "free_energy"}
    out.update({k: v[-1] for k, v in hist.items() if k != "free_energy"})
    out["free_energy"] = np.stack(hist["free_energy"])
    out["z_prob"] = np.moveaxis(r, 0, -1)                                 # [N, K, B]
    return out


def log_rho(Y, alpha, m, Vm, nu, iS):
    """log rho[b, i, k] of q(z_i) (unnormalised), Y[B, N, d]."""
    d = Y.shape[-1]
    EW = nu[..., None, None] * np.linalg.inv(iS)
    dy = Y[:, :, None, :] - m[:, None]
    quad = np.einsum("bnki,bkij,bnkj->bnk", dy, EW, dy) + np.einsum("bkij,bkji->bk", EW, Vm)[:, None]
    elogs = digamma(alpha) - digamma(alpha.sum(1, keepdims=True))
    return (elogs + 0.5 * _elogdet_w(nu, iS))[:, None] - 0.5 * d * LOG2PI - 0.5 * quad


def free_energy(Y, r, alpha, m, Vm, nu, iS, alpha0, mu0, V0, nu0, S0):
    """Bethe free energy in closed form: KL(q(s) || prior) + sum_k KL(q(m_k) || prior) + sum_k KL(q(W_k) || prior)
    + sum_i (U_Categorical,i + U_NormalMixture,i - H[q(z_i)]); the data are PointMass (no entropy).  The form the kernel
    evaluates: the NormalMixture energies through sum_i r_ik (y_i - m_k)(y_i - m_k)'."""
    d = Y.shape[-1]
    alpha0 = np.asarray(alpha0, np.float64); nu0 = np.asarray(nu0, np.float64)
    V0i = np.linalg.inv(V0); S0i = np.linalg.inv(S0)
    Nk = r.sum(1)
    sa = alpha.sum(1)
    elogs = digamma(alpha) - digamma(sa)[:, None]
    kl_s = (gammaln(sa) - gammaln(alpha).sum(1) - gammaln(alpha0.sum()) + gammaln(alpha0).sum()
            + ((alpha - alpha0) * elogs).sum(1))
    e = m - mu0[None]
    kl_m = 0.5 * (np.einsum("kij,bkji->bk", V0i, Vm) + np.einsum("bki,kij,bkj->bk", e, V0i, e) - d
                  + np.linalg.slogdet(V0)[1][None] - np.linalg.slogdet(Vm)[1])
    S = np.linalg.inv(iS)
    elw = _elogdet_w(nu, iS)
    logdetS = -np.linalg.slogdet(iS)[1]
    kl_w = (0.5 * (nu - nu0) * elw - 0.5 * nu * d + 0.5 * nu * np.einsum("kij,bkji->bk", S0i, S)
            - 0.5 * (nu - nu0) * d * np.log(2.0) - 0.5 * nu * logdetS + 0.5 * nu0 * np.linalg.slogdet(S0)[1]
            - multigammaln(0.5 * nu, d) + multigammaln(0.5 * nu0, d))
    dy = Y[:, :, None, :] - m[:, None]
    R = np.einsum("bnk,bnki,bnkj->bkij", r, dy, dy)
    EW = nu[..., None, None] * S
    U_nm = Nk * (0.5 * d * LOG2PI - 0.5 * elw) + 0.5 * np.einsum("bkij,bkji->bk", EW, R + Nk[..., None, None] * Vm)
    U_cat = -(Nk * elogs).sum(1)
    with np.errstate(divide="ignore", invalid="ignore"):
        Hz = -np.where(r > 0, r * np.log(np.where(r > 0, r, 1.0)), 0.0).sum((1, 2))
    return kl_s + kl_m.sum(1) + kl_w.sum(1) + U_cat + U_nm.sum(1) - Hz


def free_energy_dense(Y, r, alpha, m, Vm, nu, iS, alpha0, mu0, V0, nu0, S0):
    """The definition, chain by chain: sum of every node's average energy -E_q[log f] (each expectation written out
    point by point) minus the entropies of every q, the entropies from scipy."""
    B, N, d = Y.shape
    K = len(alpha0)
    out = np.zeros(B)
    for b in range(B):
        S = [np.linalg.inv(iS[b, k]) for k in range(K)]
        EW = [nu[b, k] * S[k] for k in range(K)]
        elw = [_elogdet_w(nu[b, k], iS[b, k]) for k in range(K)]
        elogs = digamma(alpha[b]) - digamma(alpha[b].sum())
        # Dirichlet prior node
        U = -(gammaln(np.sum(alpha0)) - gammaln(alpha0).sum() + ((np.asarray(alpha0) - 1) * elogs).sum())
        H = stats.dirichlet(alpha[b]).entropy()
        for k in range(K):
            # Gaussian prior on m_k: -E log N(m_k | mu0, V0)
            e = m[b, k] - mu0[k]
            U += 0.5 * (d * LOG2PI + np.linalg.slogdet(V0[k])[1] + np.trace(np.linalg.solve(V0[k], Vm[b, k] + np.outer(e, e))))
            # Wishart prior on W_k: -E log Wishart(W_k | nu0, S0)
            U -= (0.5 * (nu0[k] - d - 1) * elw[k] - 0.5 * np.trace(np.linalg.solve(S0[k], EW[k])) - 0.5 * nu0[k] * d * np.log(2)
                  - 0.5 * nu0[k] * np.linalg.slogdet(S0[k])[1] - multigammaln(0.5 * nu0[k], d))
            H += stats.multivariate_normal(m[b, k], Vm[b, k]).entropy() + stats.wishart(nu[b, k], S[k]).entropy()
        for i in range(N):
            for k in range(K):
                rik = r[b, i, k]
                e = Y[b, i] - m[b, k]
                U -= rik * elogs[k]                                           # Categorical node
                U += rik * 0.5 * (d * LOG2PI - elw[k] + e @ EW[k] @ e + np.trace(EW[k] @ Vm[b, k]))   # NormalMixture
                if rik > 0:
                    H -= rik * np.log(rik)
        out[b] = U - H
    return out


# --------------------------------------------------------------------------- problems
def random_spd(rng, d, scale=1.0):
    M = rng.standard_normal((d, d))
    return scale * (M @ M.T / d + 0.5 * np.eye(d))


def problem(d, K, N, batch, seed, radius=4.0, overlap=False):
    """Distinct data per chain: K clusters around random centres (radius ``radius``), non-trivial priors and initial
    marginals (non-identity V0 / S0, nu0 != d + 1, unequal alpha0)."""
    rng = np.random.default_rng(seed)
    y = np.zeros((N, d, batch))
    spread = 0.3 if overlap else 1.0
    for b in range(batch):
        centres = radius * spread * rng.standard_normal((K, d)) + radius * rng.standard_normal(d) * (1 - spread)
        w = rng.dirichlet(np.full(K, 3.0))
        z = rng.choice(K, size=N, p=w)
        covs = [random_spd(rng, d, 0.5 + rng.random()) for _ in range(K)]
        for i in range(N):
            y[i, :, b] = rng.multivariate_normal(centres[z[i]], covs[z[i]])
    ctr = y.mean((0, 2))
    pri = dict(alpha0=0.5 + rng.random(K),
               mu0=ctr + radius * rng.standard_normal((K, d)),
               V0=np.stack([random_spd(rng, d, 10.0 * radius ** 2) for _ in range(K)]),
               nu0=d + 0.5 + rng.random(K) * 2,
               S0=np.stack([random_spd(rng, d, 0.3) for _ in range(K)]),
               alpha_init=1.0 + rng.random(K),
               m_init=ctr + radius * rng.standard_normal((K, d)),
               Vm_init=np.stack([random_spd(rng, d, 2.0) for _ in range(K)]),
               nu_init=d + 1.0 + rng.random(K),
               S_init=np.stack([random_spd(rng, d, 0.2) for _ in range(K)]))
    return y, pri


def f32(x):
    return np.asarray(x, np.float32).astype(np.float64)


# --------------------------------------------------------------------------- the reference tests' data
# The data are replayed with the restated StableRNG (oracle/julia_rng.py).  The labels come from Distributions'
# `rand(rng, Categorical(p), n)`, whose sampler is not restated exactly; CATEGORICAL_READINGS are the candidate readings
# tried against the free-energy pins (scripts/explore_gmm_pins.py, DESIGN 3.17).  None reproduces both pins, so the
# tests use the first, the classic alias table, for data drawn from the same models.
M64 = (1 << 64) - 1


def range_ndl(rng, s):
    """rand(rng, 1:s), Julia >= 1.5: Lemire's nearly-divisionless sampler on one UInt64 (rejection on the low word)."""
    x = rng.u64(); m = x * s; lo = m & M64
    if lo < s:
        t = ((1 << 64) - s) % s
        while lo < t:
            x = rng.u64(); m = x * s; lo = m & M64
    return (m >> 64) + 1


def range_masked(rng, s):
    """rand(rng, 1:s) through a bit mask and rejection (Julia's SamplerRangeFast)."""
    mask = (1 << (s - 1).bit_length()) - 1
    while True:
        x = rng.u64() & mask
        if x <= s - 1:
            return x + 1


def alias_table(p):
    """Walker / Vose alias table as Distributions' classic `make_alias_table!` builds it: accept[i], alias[i] (1-based)."""
    n = len(p)
    w = np.asarray(p, np.float64)
    a = list(w * (n / w.sum()))
    alias = list(range(1, n + 1))
    larges = [i for i in range(n) if a[i] > 1.0]
    smalls = [i for i in range(n) if a[i] < 1.0]
    while larges and smalls:
        sm, lg = smalls.pop(), larges.pop()
        alias[sm] = lg + 1
        a[lg] = (a[lg] - 1.0) + a[sm]
        (larges if a[lg] > 1.0 else smalls).append(lg)
    for i in smalls + larges:
        a[i] = 1.0
    return a, alias


def _alias_two_draws(index):
    def draw(rng, p, n):
        a, alias = alias_table(p)
        out = []
        for _ in range(n):
            i = index(rng, len(p))
            out.append(i if rng.rand() < a[i - 1] else alias[i - 1])
        return out
    return draw


def _alias_one_draw(rng, p, n):
    """One UInt64 per label: the top bits pick one of 2^k cells, the remaining bits are the acceptance variate."""
    a, alias = alias_table(p)
    L = 1 << (len(p) - 1).bit_length()
    k = L.bit_length() - 1
    a, alias = a + [0.0] * (L - len(p)), alias + [1] * (L - len(p))
    out = []
    for _ in range(n):
        x = rng.u64()
        c = x >> (64 - k) if k else 0
        u = (x & ((1 << (64 - k)) - 1)) / float(1 << (64 - k))
        out.append(c + 1 if u < a[c] else alias[c])
    return out


def _inverse_cdf(rng, p, n):
    cp = np.cumsum(p)
    return [int(np.searchsorted(cp, rng.rand(), side="right")) + 1 for _ in range(n)]


CATEGORICAL_READINGS = {"alias, rand(1:n) nearly-divisionless + rand()": _alias_two_draws(range_ndl),
                        "alias, rand(1:n) masked + rand()": _alias_two_draws(range_masked),
                        "alias, one UInt64 per draw": _alias_one_draw,
                        "inverse cdf, one rand()": _inverse_cdf}
DEFAULT_READING = next(iter(CATEGORICAL_READINGS))


def univariate_reference_data(seed=12345, n=150, reading=DEFAULT_READING):
    """gmm_univariate_tests.jl:42-60: StableRNG(12345); z = rand(rng, Categorical([1/3, 2/3]), n), then
    y[i] = rand(rng, Normal(mu[z], 1 / sqrt(w[z]))) = mu + sigma randn(rng)."""
    from oracle.julia_rng import StableRNG
    rng = StableRNG(seed)
    switch = np.array([1 / 3, 2 / 3])
    mus, ws = np.array([-10.0, 10.0]), np.array([3.777, 0.333])
    z = CATEGORICAL_READINGS[reading](rng, list(switch), n)
    y = np.array([mus[zi - 1] + np.sqrt(1.0 / ws[zi - 1]) * rng.randn() for zi in z])
    return y, switch, mus, ws


def univariate_reference_model():
    """Priors and initialization of gmm_univariate_tests.jl:6-26 in the Dirichlet / Wishart form."""
    from rxinfer_jl_b200 import Beta, GammaShapeRate, NormalMeanVariance, vague
    from rxinfer_jl_b200.inference import gaussian_mixture as gm, gaussian_mixture_arrays
    model = gm(K=2, alpha0=Beta(1.0, 1.0), m_prior=[NormalMeanVariance(-2.0, 1e3), NormalMeanVariance(2.0, 1e3)],
               w_prior=[GammaShapeRate(0.01, 0.01), GammaShapeRate(0.01, 0.01)])
    init = {"s": vague(Beta), "m": [NormalMeanVariance(-2.0, 1e3), NormalMeanVariance(2.0, 1e3)],
            "w": [vague(GammaShapeRate), vague(GammaShapeRate)]}
    return model, init, gaussian_mixture_arrays(model, init)


def multivariate_reference_data(seed=43, n=500, L=50.0, K=3, reading=DEFAULT_READING):
    """gmm_multivariate_tests.jl:66-104 (clusters on a circle of radius L): StableRNG(43); the labels, then
    rand(rng, MvNormal(mean, cov)) = mean + cholesky(cov).L * [randn(rng), randn(rng)] per point."""
    from oracle.julia_rng import StableRNG
    rng = StableRNG(seed)
    means, chols = [], []
    for i in range(K):
        a = 2 * np.pi / K * i
        R = np.array([[np.cos(a), -np.sin(a)], [np.sin(a), np.cos(a)]])
        C = R @ np.diag([10.0, 20.0]) @ R.T
        means.append(R @ np.array([L, 0.0])); chols.append(np.linalg.cholesky(0.5 * (C + C.T)))   # Hermitian(...)
    z = CATEGORICAL_READINGS[reading](rng, [1.0 / K] * K, n)
    y = np.stack([means[zi - 1] + chols[zi - 1] @ np.array([rng.randn(), rng.randn()]) for zi in z])
    return y, np.array(means)


def multivariate_reference_model(seed=42, L=50.0, K=3):
    """Priors (gmm_multivariate_tests.jl:10-19) and initial marginals (:37-58) from the restated StableRNG(42): the same
    rng is drawn first by the initialization loop and then by the model, so prior means and initial means differ.  Per
    component: rand(rng) for the angle, rand(rng, 2) for the basis vector."""
    from oracle.julia_rng import StableRNG
    from rxinfer_jl_b200 import Dirichlet, MvNormalMeanCovariance, Wishart, vague
    from rxinfer_jl_b200.inference import gaussian_mixture as gm, gaussian_mixture_arrays
    rng = StableRNG(seed)

    def approx_means():
        out = []
        for i in range(K):
            ang = ((2 * np.pi + rng.rand()) / K) * i
            v = L / 2 * (np.array([1.0, 0.0]) + np.array([rng.rand(), rng.rand()]))
            R = np.array([[np.cos(ang), -np.sin(ang)], [np.sin(ang), np.cos(ang)]])
            out.append(R @ v)
        return out

    init_means = approx_means()
    prior_means = approx_means()
    cov = np.diag([1e6, 1e6])
    model = gm(K=K, alpha0=Dirichlet(np.ones(K)), m_prior=[MvNormalMeanCovariance(mu, cov) for mu in prior_means],
               w_prior=[Wishart(3, np.diag([1e2, 1e2])) for _ in range(K)])
    init = {"s": vague(Dirichlet, K), "m": [MvNormalMeanCovariance(mu, cov) for mu in init_means],
            "w": [Wishart(3, np.diag([1e2, 1e2])) for _ in range(K)]}
    return model, init, gaussian_mixture_arrays(model, init)


PRIOR_KEYS = ("alpha0", "mu0", "V0", "nu0", "S0", "alpha_init", "m_init", "Vm_init", "nu_init", "S_init")


def run_arrays(y, arr, iterations, **kw):
    return gaussian_mixture(y, *(arr[k] for k in PRIOR_KEYS), iterations=iterations, **kw)


def univariate_assertions(r, switch, mus, ws):
    """gmm_univariate_tests.jl:92-118 on results r of 10 iterations (chain 0)."""
    assert r["hist_alpha"].shape[0] == 10 and r["hist_m_mean"].shape[0] == 10 and r["hist_w_df"].shape[0] == 10
    fe = r["free_energy"][:, 0]
    assert len(fe) == 10 and np.all(np.diff(fe) <= 1e-10 * np.maximum(1.0, np.abs(fe[1:]))), fe
    a = r["alpha"][:, 0]
    ms = a[0] / a.sum()
    assert abs(ms - switch[0]) < 0.1 or abs(ms - switch[1]) < 0.1
    em = r["m_mean"][:, 0, 0]; ev = r["m_cov"][:, 0, 0, 0]
    o = np.argsort(em)
    for real, mu, v in zip(np.sort(mus), em[o], ev[o]):
        assert abs(real - mu) < 3 * np.sqrt(v), (real, mu, v)
    shape, rate = r["w_df"][:, 0] / 2, r["w_inv_scale"][:, 0, 0, 0] / 2
    o = np.argsort(shape / rate)
    for real, sh, rt in zip(np.sort(ws), shape[o], rate[o]):
        assert abs(real - sh / rt) < 3 * np.sqrt(sh) / rt, (real, sh / rt)


def multivariate_assertions(r, means):
    """gmm_multivariate_tests.jl:96-110 on results r of 25 iterations (chain 0)."""
    assert r["hist_alpha"].shape[0] == 25 and r["hist_m_mean"].shape[0] == 25 and r["hist_w_df"].shape[0] == 25
    fe = r["free_energy"][:, 0]
    assert len(fe) == 25
    dfe = np.diff(fe)
    assert np.all(dfe[np.abs(dfe) > 1e-3] < 0), fe
    key = lambda x: np.arctan(x[1] / x[0])
    est = sorted(list(r["m_mean"][:, :, 0]), key=key)
    real = sorted(list(means), key=key)
    for e, t in zip(est, real):
        assert np.linalg.norm(e / np.linalg.norm(e) - t / np.linalg.norm(t)) < 0.1, (e, t)


# --------------------------------------------------------------------------- tests
@pytest.mark.parametrize("d,K", [(1, 2), (1, 3), (2, 3), (2, 8), (4, 2), (4, 3), (4, 8)])
def test_closed_form_free_energy_equals_the_definition(d, K):
    y, pri = problem(d, K, 12, 2, seed=10 * d + K)
    r = gaussian_mixture(y, **pri, iterations=3)
    Y = np.moveaxis(y, 2, 0)
    args = (Y, np.moveaxis(r["z_prob"], -1, 0), r["alpha"].T, np.moveaxis(r["m_mean"], -1, 0),
            np.moveaxis(r["m_cov"], -1, 0), r["w_df"].T, np.moveaxis(r["w_inv_scale"], -1, 0), pri["alpha0"], pri["mu0"],
            pri["V0"], pri["nu0"], pri["S0"])
    closed, dense = free_energy(*args), free_energy_dense(*args)
    assert np.allclose(r["free_energy"][-1], closed, rtol=1e-13, atol=0)
    assert np.all(np.abs(closed - dense) <= 1e-10 * np.maximum(1.0, np.abs(dense))), (closed, dense)


@pytest.mark.parametrize("d,K", [(1, 2), (2, 3), (3, 5), (4, 8)])
def test_every_update_is_the_conjugate_sufficient_statistic_update(d, K):
    """Per iteration, from the oracle's own q(z): N_k = sum r, sy = sum r y, syy = sum r y y';
    q(m): Lambda = V0^-1 + N E[W] (previous), m = Lambda^-1 (V0^-1 mu0 + E[W] sy);
    q(W): nu = nu0 + N, inv_scale = inv(S0) + syy - sy m' - m sy' + N (m m' + V);  q(s): alpha0 + N."""
    y, pri = problem(d, K, 30, 3, seed=7 + d)
    its = 4
    r = gaussian_mixture(y, **pri, iterations=its)
    inv = np.linalg.inv
    for b in range(3):
        Yb = y[:, :, b]
        m, V = pri["m_init"].copy(), pri["Vm_init"].copy()
        nu, iS = pri["nu_init"].copy(), inv(pri["S_init"])
        alpha = pri["alpha_init"].copy()
        for it in range(its):
            lr = log_rho(Yb[None], alpha[None], m[None], V[None], nu[None], iS[None])[0]
            rr = np.exp(lr - logsumexp(lr, axis=1, keepdims=True))
            for k in range(K):
                Nk, sy, syy = rr[:, k].sum(), rr[:, k] @ Yb, (rr[:, k, None] * Yb).T @ Yb
                EW = nu[k] * inv(iS[k])
                V[k] = inv(inv(pri["V0"][k]) + Nk * EW)
                m[k] = V[k] @ (inv(pri["V0"][k]) @ pri["mu0"][k] + EW @ sy)
                iS[k] = inv(pri["S0"][k]) + syy - np.outer(sy, m[k]) - np.outer(m[k], sy) + Nk * (np.outer(m[k], m[k]) + V[k])
                nu[k] = pri["nu0"][k] + Nk
                alpha[k] = pri["alpha0"][k] + Nk
            assert np.allclose(r["hist_m_mean"][it, :, :, b], m, rtol=1e-9, atol=1e-9)
            assert np.allclose(r["hist_m_cov"][it, :, :, :, b], V, rtol=1e-9, atol=1e-12)
            assert np.allclose(r["hist_w_inv_scale"][it, :, :, :, b], iS, rtol=1e-9, atol=1e-9)
            assert np.allclose(r["hist_w_df"][it, :, b], nu, rtol=1e-12) and np.allclose(r["hist_alpha"][it, :, b], alpha, rtol=1e-12)


@pytest.mark.parametrize("d,K,overlap", [(1, 2, False), (2, 3, True), (3, 5, False), (4, 8, True)])
def test_free_energy_never_increases(d, K, overlap):
    y, pri = problem(d, K, 80, 4, seed=3 * d + K, overlap=overlap)
    for schedule in ("z_m_w_s", "z_w_m_s"):                 # coordinate descent on F: every step is a minimiser
        fe = gaussian_mixture(y, **pri, iterations=15, schedule=schedule)["free_energy"]
        assert np.all(np.diff(fe, axis=0) <= 1e-9 * np.abs(fe[1:])), (schedule, np.diff(fe, axis=0).max())


def scalar_beta_gamma_vmp(y, a0, b0, mu0, v0, g_shape0, g_rate0, s_init, m_init, v_init, gs_init, gr_init, iterations):
    """The univariate model written with Beta, Normal and Gamma(shape, rate) directly (one chain, y[N]):
    q(z_i = 1) from E[log s], E[log(1 - s)], E[log p_k], E[p_k] ((y - m_k)^2 + v_k); Normal / Gamma / Beta conjugate
    updates in the order q(m), q(p), q(s); free energy with Beta / Normal / Gamma entropies from scipy."""
    sa, sb = s_init
    m, v = np.array(m_init, float), np.array(v_init, float)
    gs, gr = np.array(gs_init, float), np.array(gr_init, float)
    fes = []
    for _ in range(iterations):
        el = np.array([digamma(sa), digamma(sb)]) - digamma(sa + sb)
        lr = el[None] + 0.5 * (digamma(gs) - np.log(gr))[None] - 0.5 * LOG2PI - 0.5 * (gs / gr)[None] * ((y[:, None] - m[None]) ** 2 + v[None])
        r = np.exp(lr - logsumexp(lr, axis=1, keepdims=True))
        Nk = r.sum(0)
        for k in range(2):
            prec = 1 / v0[k] + Nk[k] * gs[k] / gr[k]
            v[k] = 1 / prec
            m[k] = v[k] * (mu0[k] / v0[k] + gs[k] / gr[k] * (r[:, k] @ y))
            gs[k] = g_shape0[k] + Nk[k] / 2
            gr[k] = g_rate0[k] + 0.5 * (r[:, k] @ ((y - m[k]) ** 2) + Nk[k] * v[k])
        sa, sb = a0 + Nk[0], b0 + Nk[1]
        el = np.array([digamma(sa), digamma(sb)]) - digamma(sa + sb)
        elp = digamma(gs) - np.log(gr)
        U = -(gammaln(a0 + b0) - gammaln(a0) - gammaln(b0) + (a0 - 1) * el[0] + (b0 - 1) * el[1])
        H = stats.beta(sa, sb).entropy()
        for k in range(2):
            U += 0.5 * (LOG2PI + np.log(v0[k]) + (v[k] + (m[k] - mu0[k]) ** 2) / v0[k])
            U -= g_shape0[k] * np.log(g_rate0[k]) - gammaln(g_shape0[k]) + (g_shape0[k] - 1) * elp[k] - g_rate0[k] * gs[k] / gr[k]
            H += stats.norm(m[k], np.sqrt(v[k])).entropy() + stats.gamma(gs[k], scale=1 / gr[k]).entropy()
        U += -(r @ el).sum() + (r * (0.5 * LOG2PI - 0.5 * elp[None] + 0.5 * (gs / gr)[None] * ((y[:, None] - m[None]) ** 2 + v[None]))).sum()
        H += -(r * np.log(np.where(r > 0, r, 1.0))).sum()
        fes.append(U - H)
    return dict(s=(sa, sb), m=m, v=v, shape=gs, rate=gr, free_energy=np.array(fes))


def test_beta_gamma_spelling_equals_the_dirichlet_wishart_spelling():
    y, *_ = univariate_reference_data(seed=5, n=60)
    model, init, arr = univariate_reference_model()
    # non-default Beta / Gamma values too, through the same conversion
    from rxinfer_jl_b200 import Beta, GammaShapeRate, NormalMeanVariance
    from rxinfer_jl_b200.inference import gaussian_mixture as gm, gaussian_mixture_arrays
    model2 = gm(K=2, alpha0=Beta(2.0, 0.7), m_prior=[NormalMeanVariance(-1.0, 50.0), NormalMeanVariance(3.0, 20.0)],
                w_prior=[GammaShapeRate(1.5, 2.0), GammaShapeRate(0.4, 0.3)])
    init2 = {"s": Beta(1.3, 2.2), "m": [NormalMeanVariance(-4.0, 9.0), NormalMeanVariance(5.0, 4.0)],
             "w": [GammaShapeRate(2.0, 3.0), GammaShapeRate(1.0, 0.5)]}
    for mdl, ini, ar in ((model, init, arr), (model2, init2, gaussian_mixture_arrays(model2, init2))):
        r = run_arrays(y[:, None, None], ar, 8)
        s = scalar_beta_gamma_vmp(y, mdl.alpha0.a, mdl.alpha0.b, [x.m for x in mdl.m_prior], [x.v for x in mdl.m_prior],
                                  [x.a for x in mdl.w_prior], [x.b for x in mdl.w_prior], (ini["s"].a, ini["s"].b),
                                  [x.m for x in ini["m"]], [x.v for x in ini["m"]], [x.a for x in ini["w"]],
                                  [x.b for x in ini["w"]], 8)
        assert ar["univariate"]
        assert np.allclose(r["alpha"][:, 0], s["s"], rtol=1e-10)
        assert np.allclose(r["m_mean"][:, 0, 0], s["m"], rtol=1e-9, atol=1e-9)
        assert np.allclose(r["m_cov"][:, 0, 0, 0], s["v"], rtol=1e-9)
        assert np.allclose(r["w_df"][:, 0] / 2, s["shape"], rtol=1e-12)
        assert np.allclose(r["w_inv_scale"][:, 0, 0, 0] / 2, s["rate"], rtol=1e-9)
        assert np.allclose(r["free_energy"][:, 0], s["free_energy"], rtol=1e-10, atol=1e-8)


def test_alias_table_and_range_samplers():
    """The classic alias table of the two reference switches, and rand(1:s) within range for both range samplers."""
    from oracle.julia_rng import StableRNG
    a, alias = alias_table([1 / 3, 2 / 3])
    assert np.allclose(a, [2 / 3, 1.0]) and alias == [2, 2]
    a, alias = alias_table([1 / 3] * 3)
    assert a == [1.0, 1.0, 1.0] and alias == [1, 2, 3]
    rng = StableRNG(7)
    for s in (2, 3, 5):
        for f in (range_ndl, range_masked):
            draws = [f(rng, s) for _ in range(300)]
            assert min(draws) == 1 and max(draws) == s
    for reading, draw in CATEGORICAL_READINGS.items():
        z = np.array(draw(StableRNG(3), [1 / 3, 2 / 3], 3000))
        assert abs((z == 1).mean() - 1 / 3) < 0.03, reading


def test_univariate_reference_assertions_on_the_oracle():
    y, switch, mus, ws = univariate_reference_data()
    _, _, arr = univariate_reference_model()
    univariate_assertions(run_arrays(y[:, None, None], arr, 10), switch, mus, ws)


def test_multivariate_reference_assertions_on_the_oracle():
    y, means = multivariate_reference_data()
    _, _, arr = multivariate_reference_model()
    multivariate_assertions(run_arrays(y[:, :, None], arr, 25), means)


def test_oracle_is_translation_invariant():
    """Shifting the data and every location parameter by 1e4 leaves the oracle's posteriors (means shifted) and free
    energy unchanged.  This checks the oracle, which forms y - E[m_k] directly; the kernel's accumulation around the
    previous E[m_k] is checked on the GPU (test_mixture_gpu.py, clusters at radius 50)."""
    y, pri = problem(2, 3, 200, 2, seed=4)
    shift = np.array([1e4, -1e4])
    pri2 = dict(pri, mu0=pri["mu0"] + shift, m_init=pri["m_init"] + shift)
    r1 = gaussian_mixture(y, **pri, iterations=10)
    r2 = gaussian_mixture(y + shift[None, :, None], **pri2, iterations=10)
    assert np.allclose(r2["m_mean"] - shift[None, :, None], r1["m_mean"], atol=1e-7)
    assert np.allclose(r2["w_inv_scale"], r1["w_inv_scale"], rtol=1e-8)
    assert np.allclose(r2["free_energy"], r1["free_energy"], rtol=1e-10)


def test_host_conversion_and_argument_handling(rx):
    from rxinfer_jl_b200 import Beta, Dirichlet, GammaShapeRate, MvNormalMeanCovariance, NormalMeanVariance, Wishart, vague
    from rxinfer_jl_b200.inference import (BetheFactorization, MeanField, check_mean_field, gaussian_mixture as gm,
                                           gaussian_mixture_arrays)
    _, _, arr = univariate_reference_model()
    assert np.allclose(arr["nu0"], [0.02, 0.02]) and np.allclose(arr["S0"][:, 0, 0], [50.0, 50.0])
    assert np.allclose(arr["nu_init"], [2.0, 2.0]) and np.allclose(arr["S_init"][:, 0, 0], [0.5e12, 0.5e12])
    assert np.allclose(arr["alpha0"], [1, 1]) and np.allclose(arr["alpha_init"], [1, 1])
    assert np.allclose(vague(Dirichlet, 4).alpha, np.ones(4))
    with pytest.raises(TypeError):
        vague(Dirichlet)
    # the reference refuses every factorisation but the naive mean-field (gmm_univariate_tests.jl:117-124)
    for c in (None, BetheFactorization()):
        with pytest.raises(ValueError, match="must be the naive mean-field"):
            check_mean_field(c)
    check_mean_field(MeanField())
    model = gm(K=3, alpha0=Beta(1.0, 1.0), m_prior=[NormalMeanVariance(0.0, 1.0)] * 3, w_prior=[GammaShapeRate(1.0, 1.0)] * 3)
    init = {"s": Dirichlet(np.ones(3)), "m": [NormalMeanVariance(0.0, 1.0)] * 3, "w": [GammaShapeRate(1.0, 1.0)] * 3}
    with pytest.raises(ValueError, match="K = 2"):
        gaussian_mixture_arrays(model, init)
    model = gm(K=2, alpha0=Dirichlet(np.ones(2)), m_prior=[MvNormalMeanCovariance(np.zeros(2), np.eye(2))] * 2,
               w_prior=[Wishart(3, np.eye(2))] * 2)
    with pytest.raises(ValueError, match="initialization"):
        gaussian_mixture_arrays(model, None)
    with pytest.raises(ValueError, match="marginals for K = 2"):
        gaussian_mixture_arrays(model, {"s": Dirichlet(np.ones(2)), "m": [MvNormalMeanCovariance(np.zeros(2), np.eye(2))],
                                        "w": [Wishart(3, np.eye(2))] * 2})
    with pytest.raises(TypeError, match="Wishart or GammaShapeRate"):
        gaussian_mixture_arrays(model, {"s": Dirichlet(np.ones(2)), "m": [MvNormalMeanCovariance(np.zeros(2), np.eye(2))] * 2,
                                        "w": [np.eye(2)] * 2})
    import torch
    if not torch.cuda.is_available():
        # infer refuses a non-mean-field call before it needs a device, and needs one otherwise (no CPU fallback)
        init = {"s": Dirichlet(np.ones(2)), "m": [MvNormalMeanCovariance(np.zeros(2), np.eye(2))] * 2,
                "w": [Wishart(3, np.eye(2))] * 2}
        with pytest.raises(ValueError, match="must be the naive mean-field"):
            rx.infer(model=model, data={"y": torch.zeros(5, 2, 3)}, initialization=init, iterations=2,
                     constraints=BetheFactorization(), context=object())
        with pytest.raises(Exception):
            rx.infer(model=model, data={"y": torch.zeros(5, 2, 3)}, initialization=init, iterations=2,
                     constraints=MeanField())
        with pytest.raises(NotImplementedError):          # constraints stay refused for every other model
            rx.infer(model=rx.hgf(), data={"y": torch.zeros(5, 3)}, constraints=MeanField())
