"""Hidden Markov model with Gaussian emissions, structured VMP q(s_0, s) q(A) prod_k q(m_k) q(W_k), on the CPU.

This module holds the fp64 reference the CUDA kernel (csrc/rxg_hmm_gauss.cuh) is gated against:
  A ~ DirichletCollection(alpha_A0)   K x K, column j = p(s_t | s_{t-1} = j)  (or a known probability matrix)
  m[k] ~ MvNormal(mu0[k], V0[k]);  W[k] ~ Wishart(nu0[k], S0[k])
  s_0 ~ Categorical(p0);  s[t] ~ DiscreteTransition(s[t-1], A);  y[t] ~ NormalMixture(switch = s[t], m, W)
No reference test runs this model, so nothing pins it; the checks are against exact enumeration, the free energy's dense
definition and the model's own structure: the sweep against every path of the tilted chain, the closed-form free energy
against its definition, each update against its conjugate update from the data, the monotone free energy, translation
invariance, the univariate spelling, recovery of simulated series, the kernel body compiled for the host
(tests/c/hmm_gauss_host_harness.cu) and the host-side argument handling."""
import ctypes
import itertools
import os
import shutil
import subprocess

import numpy as np
import pytest
from scipy import stats
from scipy.special import multigammaln

from test_hmm import MISSING, _xlogy, dense_free_energy, elog_dir, kl_dir
from test_mixture import _elogdet_w, random_spd

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LOG2PI = np.log(2 * np.pi)
EMISSION_KEYS = ("mu0", "V0", "nu0", "S0", "m_init", "Vm_init", "nu_init", "S_init")


def log_weights(Y, m, Vm, nu, iS):
    """l[b, t, k] = 1/2 E log|W_k| - d/2 log 2 pi - 1/2 [(y_t - m_k)' E[W_k] (y_t - m_k) + tr(E[W_k] V_k)].
    Y[b, T, d]; m[b, K, d], Vm[b, K, d, d], nu[b, K], iS[b, K, d, d]."""
    d = Y.shape[-1]
    EW = nu[..., None, None] * np.linalg.inv(iS)
    dy = Y[:, :, None, :] - m[:, None]
    quad = np.einsum("btki,bkij,btkj->btk", dy, EW, dy) + np.einsum("bkij,bkji->bk", EW, Vm)[:, None]
    return 0.5 * _elogdet_w(nu, iS)[:, None] - 0.5 * d * LOG2PI - 0.5 * quad


def sweep(L, obs, p0, At, pairs=False):
    """Scaled forward-backward of every chain with log emission weights L[b, t, k] (ignored where obs[b, t] is False) and
    At[K, K, b].  Returns gamma[T, K, b], gamma0[K, b], xi[K, K, b], log Z~ [b] and, with ``pairs``, pair[T, K, K, b]."""
    nb, T, K = L.shape
    mx = np.where(obs, L.max(2), 0.0)                                  # [b, T]
    e = np.where(obs[..., None], np.exp(L - mx[..., None]), 1.0).transpose(1, 2, 0)   # [T, K, b]
    alpha = np.zeros((T + 1, K, nb))
    alpha[0] = p0[:, None]
    logZ = mx.sum(1)
    for t in range(1, T + 1):
        a = np.einsum("ijb,jb->ib", At, alpha[t - 1]) * e[t - 1]
        c = a.sum(0)
        alpha[t] = a / c
        logZ += np.log(c)
    beta = np.ones((K, nb))
    gamma = np.zeros((T + 1, K, nb))
    gamma[T] = alpha[T]
    xi = np.zeros((K, K, nb))
    pair = np.zeros((T, K, K, nb)) if pairs else None
    for t in range(T, 0, -1):
        w = e[t - 1] * beta
        p = At * w[:, None, :] * alpha[t - 1][None, :, :]
        p /= p.sum((0, 1))
        xi += p
        if pairs:
            pair[t - 1] = p
        gamma[t - 1] = p.sum(0)
        beta = np.einsum("ijb,ib->jb", At, w)
        beta /= (alpha[t - 1] * beta).sum(0)
    return dict(gamma=gamma[1:], gamma0=gamma[0], xi=xi, logZ=logZ, pair=pair)


def _observed(Y):
    """A step is observed when all its components are finite (an all-NaN step is missing; the kernel also reads any other
    non-finite step as missing, after flagging the chain)."""
    return np.isfinite(Y).all(-1)


def kl_normal(m, Vm, mu0, V0):
    d = m.shape[-1]
    V0i = np.linalg.inv(V0)
    e = m - mu0[None]
    return 0.5 * (np.einsum("kij,bkji->bk", V0i, Vm) + np.einsum("bki,kij,bkj->bk", e, V0i, e) - d
                  + np.linalg.slogdet(V0)[1][None] - np.linalg.slogdet(Vm)[1])


def kl_wishart(nu, iS, nu0, S0):
    d = iS.shape[-1]
    S = np.linalg.inv(iS)
    elw = _elogdet_w(nu, iS)
    return (0.5 * (nu - nu0) * elw - 0.5 * nu * d + 0.5 * nu * np.einsum("kij,bkji->bk", np.linalg.inv(S0), S)
            - 0.5 * (nu - nu0) * d * np.log(2.0) + 0.5 * nu * np.linalg.slogdet(iS)[1] + 0.5 * nu0 * np.linalg.slogdet(S0)[1]
            - multigammaln(0.5 * nu, d) + multigammaln(0.5 * nu0, d))


def hmm_gauss_vmp(y, p0, mu0, V0, nu0, S0, m_init, Vm_init, nu_init, S_init, A_prior=None, A_init=None, A_known=None,
                  iterations=1, dense=False):
    """fp64 structured VMP of every chain.  y[T, d, batch] (an all-NaN step is missing).  Per iteration: the sweep with the
    previous q(A), q(m), q(W); q(A) = Dirichlet(alpha_A0 + sum xi); q(m_k) with the previous E[W_k]; q(W_k) with the new
    q(m_k).  The Gaussian statistics are taken around the centre the sweep used, c_k = E[m_k], as the kernel does.
    Returns the kernel's outputs (s_prob[T, K, b], s0_prob, A_alpha[K, K, b] or None, m_mean[K, d, b], m_cov[K, d, d, b],
    w_df[K, b], w_inv_scale[K, d, d, b], free_energy[its, b], hist_*), the last sweep's statistics and, with ``dense``,
    free_energy_dense (the definition, term by term)."""
    y = np.asarray(y, np.float64)
    T, d, nb = y.shape
    Y = np.moveaxis(y, 2, 0)                                           # [b, T, d]
    obs = _observed(Y)
    Yz = np.where(obs[..., None], Y, 0.0)
    p0 = np.asarray(p0, np.float64)
    K = p0.shape[0]
    f = lambda v: np.asarray(v, np.float64)
    mu0, V0, nu0, S0 = f(mu0), f(V0), f(nu0), f(S0)
    V0i, S0i = np.linalg.inv(V0), np.linalg.inv(S0)
    m = np.tile(f(m_init), (nb, 1, 1))
    Vm = np.tile(f(Vm_init), (nb, 1, 1, 1))
    nu = np.tile(f(nu_init), (nb, 1))
    iS = np.tile(np.linalg.inv(f(S_init)), (nb, 1, 1, 1))
    learn_A = A_known is None
    A0 = f(A_prior) if learn_A else None
    qA = np.repeat(f(A_init)[..., None], nb, -1) if learn_A else None
    Ak = None if learn_A else np.repeat(f(A_known)[..., None], nb, -1)
    hist = {k: [] for k in ("free_energy", "free_energy_dense", "hist_s", "hist_A", "hist_m_mean", "hist_m_cov",
                            "hist_w_df", "hist_w_inv_scale")}
    for _ in range(iterations):
        A_used = elog_dir(qA) if learn_A else None
        At = np.exp(A_used) if learn_A else Ak
        L = log_weights(Yz, m, Vm, nu, iS)
        st = sweep(L, obs, p0, At, pairs=dense)
        g = np.where(obs.T[:, None, :], st["gamma"], 0.0).transpose(2, 0, 1)     # [b, T, K], 0 on missing steps
        S_used = (g * L).sum((1, 2))
        # statistics around the centre the sweep used
        c = m.copy()
        EWp = nu[..., None, None] * np.linalg.inv(iS)
        dy = Yz[:, :, None, :] - c[:, None]                                        # [b, T, K, d]
        N = g.sum(1)
        bk = np.einsum("btk,btki->bki", g, dy)
        Ck = np.einsum("btk,btki,btkj->bkij", g, dy, dy)
        # updates
        if learn_A:
            qA = A0[..., None] + st["xi"]
        Vm = np.linalg.inv(V0i[None] + N[..., None, None] * EWp)
        xi = np.einsum("kij,kj->ki", V0i, mu0)[None] + np.einsum("bkij,bkj->bki", EWp, bk + N[..., None] * c)
        m = np.einsum("bkij,bkj->bki", Vm, xi)
        dm = m - c
        R = (Ck - np.einsum("bki,bkj->bkij", bk, dm) - np.einsum("bki,bkj->bkij", dm, bk)
             + N[..., None, None] * np.einsum("bki,bkj->bkij", dm, dm))
        nu = nu0[None] + N
        iS = S0i[None] + R + N[..., None, None] * Vm
        # closed-form free energy
        EW = nu[..., None, None] * np.linalg.inv(iS)
        elw = _elogdet_w(nu, iS)
        F = -st["logZ"] + S_used
        if learn_A:
            F += kl_dir(qA, A0) + (st["xi"] * (A_used - elog_dir(qA))).sum((0, 1))
        F += (kl_normal(m, Vm, mu0, V0) + kl_wishart(nu, iS, nu0, S0) + N * (0.5 * d * LOG2PI - 0.5 * elw)
              + 0.5 * np.einsum("bkij,bkji->bk", EW, R + N[..., None, None] * Vm)).sum(1)
        hist["free_energy"].append(F)
        if dense:
            hist["free_energy_dense"].append(free_energy_dense(Yz, obs, p0, st, A0, qA, Ak, m, Vm, nu, iS, mu0, V0, nu0, S0))
        hist["hist_s"].append(st["gamma"])
        hist["hist_A"].append(qA)
        hist["hist_m_mean"].append(np.moveaxis(m, 0, -1))
        hist["hist_m_cov"].append(np.moveaxis(Vm, 0, -1))
        hist["hist_w_df"].append(nu.T.copy())
        hist["hist_w_inv_scale"].append(np.moveaxis(iS, 0, -1))
    out = {k: np.stack(v) for k, v in hist.items() if v and v[0] is not None}
    out["hist_A"] = out.get("hist_A")
    out.update(s_prob=st["gamma"], s0_prob=st["gamma0"], A_alpha=qA, m_mean=out["hist_m_mean"][-1],
               m_cov=out["hist_m_cov"][-1], w_df=out["hist_w_df"][-1], w_inv_scale=out["hist_w_inv_scale"][-1],
               xi=st["xi"], pair=st["pair"], logZ=st["logZ"])
    return out


def free_energy_dense(Yz, obs, p0, st, A0, qA, Ak, m, Vm, nu, iS, mu0, V0, nu0, S0):
    """E_q[-log p(y, s_0, s, A, m, W)] - H[q(s_0, s)] - H[q(A)] - sum H[q(m_k)] - sum H[q(W_k)], term by term: the chain and A
    terms as test_hmm.dense_free_energy (no symbol emissions), the emissions -sum gamma_tk E log N(y_t | m_k, inv(W_k))
    point by point, the Gaussian and Wishart priors and entropies chain by chain (entropies from scipy)."""
    nb, T, d = Yz.shape
    K = p0.shape[0]
    F = dense_free_energy(np.full((T, nb), MISSING), p0, st, A0, qA, Ak, None, None, None)
    L_new = log_weights(Yz, m, Vm, nu, iS)                             # E_q log N(y_t | m_k, inv(W_k)) with the new q
    g = st["gamma"].transpose(2, 0, 1)
    F -= np.where(obs[..., None], g * L_new, 0.0).sum((1, 2))
    for b in range(nb):
        for k in range(K):
            S = np.linalg.inv(iS[b, k])
            EW = nu[b, k] * S
            elw = _elogdet_w(nu[b, k], iS[b, k])
            e = m[b, k] - mu0[k]
            U = 0.5 * (d * LOG2PI + np.linalg.slogdet(V0[k])[1] + np.trace(np.linalg.solve(V0[k], Vm[b, k] + np.outer(e, e))))
            U -= (0.5 * (nu0[k] - d - 1) * elw - 0.5 * np.trace(np.linalg.solve(S0[k], EW)) - 0.5 * nu0[k] * d * np.log(2)
                  - 0.5 * nu0[k] * np.linalg.slogdet(S0[k])[1] - multigammaln(0.5 * nu0[k], d))
            H = stats.multivariate_normal(m[b, k], Vm[b, k]).entropy() + stats.wishart(nu[b, k], S).entropy()
            F[b] += U - H
    return F


# --------------------------------------------------------------------------- problems
def random_problem(d, K, T, nb, seed, learn_A=True, p_missing=0.0, sharp=False, radius=4.0, offset=0.0):
    """Distinct series per chain drawn from a random model (K well-spread means, random covariances), priors and initial
    marginals shared by every chain (non-identity V0 / S0, nu0 != d + 1, non-symmetric Dirichlet parameters), or the
    known A; a fraction ``p_missing`` of all-NaN steps."""
    rng = np.random.default_rng(seed)
    A = rng.dirichlet(np.full(K, 0.5), K).T
    A = 0.999 * np.eye(K) + 0.001 * A if sharp else 0.5 * np.eye(K) + 0.5 * A
    p0 = rng.dirichlet(np.ones(K))
    y = np.zeros((T, d, nb))
    for b in range(nb):
        centres = offset + radius * rng.standard_normal((K, d))
        chol = [np.linalg.cholesky(random_spd(rng, d, 0.3 + 0.5 * rng.random())) for _ in range(K)]
        s = rng.choice(K, p=p0)
        for t in range(T):
            s = rng.choice(K, p=A[:, s])
            y[t, :, b] = centres[s] + chol[s] @ rng.standard_normal(d)
    miss = rng.random((T, nb)) < p_missing
    y[np.repeat(miss[:, None, :], d, 1)] = np.nan
    kw = dict(p0=p0, mu0=offset + radius * rng.standard_normal((K, d)),
              V0=np.stack([random_spd(rng, d, 10.0 * radius ** 2) for _ in range(K)]), nu0=d + 0.5 + 2 * rng.random(K),
              S0=np.stack([random_spd(rng, d, 0.3) for _ in range(K)]), m_init=offset + radius * rng.standard_normal((K, d)),
              Vm_init=np.stack([random_spd(rng, d, 2.0) for _ in range(K)]), nu_init=d + 1.0 + rng.random(K),
              S_init=np.stack([random_spd(rng, d, 0.2) for _ in range(K)]))
    if learn_A:
        kw.update(A_prior=rng.uniform(0.3, 3.0, (K, K)), A_init=rng.uniform(0.5, 4.0, (K, K)) + 3 * np.eye(K))
    else:
        kw.update(A_known=A)
    return y, kw


def f32(a):
    return None if a is None else np.asarray(a, np.float32).astype(np.float64)


def reference_on_f32(y, kw, iterations):
    return hmm_gauss_vmp(f32(y), **{k: f32(v) for k, v in kw.items()}, iterations=iterations)


def brute_force(L, obs, p0, A):
    """q(s_t), q(s_{t-1}, s_t) and log Z~ of one chain by summing over all K^(T+1) paths of p0 prod A prod exp(l(y_t))."""
    T, K = L.shape[0], len(p0)
    paths = list(itertools.product(range(K), repeat=T + 1))
    lp = np.array([np.log(p0[s[0]]) + sum(np.log(A[s[t + 1], s[t]]) + (L[t, s[t + 1]] if obs[t] else 0.0)
                                          for t in range(T)) for s in paths])
    logZ = np.log(np.exp(lp - lp.max()).sum()) + lp.max()
    w = np.exp(lp - logZ)
    gamma, pair = np.zeros((T, K)), np.zeros((T, K, K))
    for s, wi in zip(paths, w):
        for t in range(T):
            gamma[t, s[t + 1]] += wi
            pair[t, s[t + 1], s[t]] += wi
    return gamma, pair, logZ


# --------------------------------------------------------------------------- the reference against independent computations
@pytest.mark.parametrize("T,p_missing", [(1, 0.0), (4, 0.0), (6, 0.0), (6, 0.4)])
def test_one_sweep_equals_enumeration_of_the_tilted_model(T, p_missing):
    for learn_A in (True, False):
        y, kw = random_problem(2, 3, T, 3, seed=T + int(10 * p_missing) + 7 * learn_A, learn_A=learn_A, p_missing=p_missing)
        if p_missing:
            y[2, :, 0] = np.nan
        r = hmm_gauss_vmp(y, **kw, iterations=1, dense=True)
        Y = np.moveaxis(y, 2, 0)
        obs = _observed(Y)
        nb = y.shape[2]
        m, Vm = np.tile(kw["m_init"], (nb, 1, 1)), np.tile(kw["Vm_init"], (nb, 1, 1, 1))
        nu, iS = np.tile(kw["nu_init"], (nb, 1)), np.tile(np.linalg.inv(kw["S_init"]), (nb, 1, 1, 1))
        L = log_weights(np.where(obs[..., None], Y, 0.0), m, Vm, nu, iS)
        A = np.exp(elog_dir(kw["A_init"])) if learn_A else kw["A_known"]
        for b in range(nb):
            g, pair, logZ = brute_force(L[b], obs[b], kw["p0"], A)
            assert np.abs(r["s_prob"][:, :, b] - g).max() < 1e-12
            assert np.abs(r["pair"][..., b] - pair).max() < 1e-12
            assert abs(r["logZ"][b] - logZ) < 1e-12 * max(1.0, abs(logZ))


@pytest.mark.parametrize("learn_A", [True, False])
@pytest.mark.parametrize("d,K", [(1, 2), (2, 3), (3, 5), (4, 8)])
def test_closed_form_free_energy_equals_the_definition(d, K, learn_A):
    y, kw = random_problem(d, K, 12, 3, seed=10 * d + K, learn_A=learn_A, p_missing=0.2)
    r = hmm_gauss_vmp(y, **kw, iterations=4, dense=True)
    assert np.abs(r["free_energy"] - r["free_energy_dense"]).max() < 1e-10


@pytest.mark.parametrize("d,K", [(1, 2), (2, 3), (3, 5), (4, 8)])
def test_every_update_is_its_conjugate_update_from_the_data(d, K):
    """One iteration: q(A) = alpha_A0 + sum xi; q(m_k) = prior x prod_t N(y_t | m_k, (gamma_tk E[W_k])^-1);
    q(W_k) = Wishart(nu0 + N_k, inv(inv(S0) + sum_t gamma_tk ((y_t - m)(y_t - m)' + V_k))), from gamma, xi and the data
    directly (no statistics around a centre)."""
    y, kw = random_problem(d, K, 25, 3, seed=40 + d, p_missing=0.2)
    r = hmm_gauss_vmp(y, **kw, iterations=1)
    Y = np.moveaxis(y, 2, 0)
    obs = _observed(Y)
    Yz = np.where(obs[..., None], Y, 0.0)
    nb = y.shape[2]
    EW0 = kw["nu_init"][:, None, None] * kw["S_init"]                                      # E[W_k], [K, d, d]
    g = np.where(obs.T[:, None, :], r["s_prob"], 0.0)                                      # [T, K, b]
    st = sweep(log_weights(Yz, np.tile(kw["m_init"], (nb, 1, 1)), np.tile(kw["Vm_init"], (nb, 1, 1, 1)),
                           np.tile(kw["nu_init"], (nb, 1)), np.tile(np.linalg.inv(kw["S_init"]), (nb, 1, 1, 1))),
               obs, kw["p0"], np.repeat(np.exp(elog_dir(kw["A_init"]))[..., None], nb, -1), pairs=True)
    assert np.abs(r["A_alpha"] - (kw["A_prior"][..., None] + st["pair"].sum(0))).max() < 1e-12
    assert np.abs(r["s_prob"] - st["pair"].sum(2)).max() < 1e-12
    V0i = np.linalg.inv(kw["V0"])
    for b in range(nb):
        for k in range(K):
            gk = g[:, k, b]
            P = V0i[k] + gk.sum() * EW0[k]
            Vm = np.linalg.inv(P)
            m = Vm @ (V0i[k] @ kw["mu0"][k] + EW0[k] @ (gk[:, None] * Yz[b]).sum(0))
            assert np.allclose(r["m_cov"][k, :, :, b], Vm, rtol=1e-10, atol=1e-12)
            assert np.allclose(r["m_mean"][k, :, b], m, rtol=1e-10, atol=1e-10)
            dy = Yz[b] - m
            iS = np.linalg.inv(kw["S0"][k]) + np.einsum("t,ti,tj->ij", gk, dy, dy) + gk.sum() * Vm
            assert abs(r["w_df"][k, b] - (kw["nu0"][k] + gk.sum())) < 1e-10
            assert np.allclose(r["w_inv_scale"][k, :, :, b], iS, rtol=1e-10, atol=1e-10)


@pytest.mark.parametrize("learn_A", [True, False])
@pytest.mark.parametrize("d,K", [(1, 2), (2, 3), (3, 5), (4, 8)])
def test_free_energy_never_increases(d, K, learn_A):
    y, kw = random_problem(d, K, 60, 3, seed=60 + d + K, learn_A=learn_A, p_missing=0.1)
    fe = hmm_gauss_vmp(y, **kw, iterations=25)["free_energy"]
    assert np.all(np.diff(fe, axis=0) <= 1e-9 * np.maximum(np.abs(fe[:-1]), 1.0))


def test_a_shift_of_the_data_and_the_means_leaves_the_posteriors_and_f_unchanged():
    y, kw = random_problem(2, 3, 40, 3, seed=77, p_missing=0.1)
    r = hmm_gauss_vmp(y, **kw, iterations=8)
    shift = 1e4 * np.array([1.0, -0.7])
    ks = dict(kw, mu0=kw["mu0"] + shift, m_init=kw["m_init"] + shift)
    rs = hmm_gauss_vmp(y + shift[None, :, None], **ks, iterations=8)
    assert np.abs(rs["m_mean"] - shift[None, :, None] - r["m_mean"]).max() < 1e-6
    for k in ("s_prob", "A_alpha", "m_cov", "w_df", "w_inv_scale"):
        assert np.abs(rs[k] - r[k]).max() < 1e-6 * max(1.0, np.abs(r[k]).max()), k
    assert np.abs(rs["free_energy"] - r["free_energy"]).max() < 1e-7 * np.abs(r["free_energy"]).max()


# --------------------------------------------------------------------------- recovery
def recovery_problem(nb=1, seed=2024, T=1000):
    """K = 3, d = 2, 0.9 on the diagonal of A; means (0, 0), (4, 0), (0, 4); initial means perturbed from the truth."""
    rng = np.random.default_rng(seed)
    K, d = 3, 2
    A = np.full((K, K), 0.05) + 0.85 * np.eye(K)
    means = np.array([[0.0, 0.0], [4.0, 0.0], [0.0, 4.0]])
    covs = [random_spd(rng, d, 0.6) for _ in range(K)]
    y, s_true = np.zeros((T, d, nb)), np.zeros((T, nb), int)
    for b in range(nb):
        s = rng.integers(K)
        for t in range(T):
            s = rng.choice(K, p=A[:, s])
            s_true[t, b] = s
            y[t, :, b] = rng.multivariate_normal(means[s], covs[s])
    kw = dict(p0=np.full(K, 1 / K), A_prior=np.ones((K, K)), A_init=np.ones((K, K)) + 4 * np.eye(K),
              mu0=np.zeros((K, d)), V0=np.stack([100.0 * np.eye(d)] * K), nu0=np.full(K, d + 2.0),
              S0=np.stack([np.eye(d) / (d + 2.0)] * K), m_init=means + rng.uniform(-1.0, 1.0, (K, d)),
              Vm_init=np.stack([np.eye(d)] * K), nu_init=np.full(K, d + 2.0), S_init=np.stack([np.eye(d) / (d + 2.0)] * K))
    return y, s_true, means, A, kw


def recovery_assertions(r, s_true, means, A, b=0):
    """After label matching: E[m_k] within 0.3, the diagonal of E[A] within 0.05, argmax q(s_t) right on >= 95 % of steps."""
    K = means.shape[0]
    mm = np.asarray(r["m_mean"], np.float64)[..., b]                    # [K, d]
    perm = min(itertools.permutations(range(K)), key=lambda p: np.abs(mm[list(p)] - means).sum())
    assert np.abs(mm[list(perm)] - means).max() < 0.3
    al = np.asarray(r["A_alpha"], np.float64)[..., b]
    EA = al / al.sum(0, keepdims=True)
    assert np.abs(np.diag(EA)[list(perm)] - np.diag(A)).max() < 0.05
    inv = np.argsort(perm)                                              # estimated label -> true label
    s_hat = inv[np.asarray(r["s_prob"], np.float64)[:, :, b].argmax(1)]
    assert np.mean(s_hat == s_true[:, b]) >= 0.95


def test_recovery_on_series_drawn_from_the_model():
    y, s_true, means, A, kw = recovery_problem()
    r = hmm_gauss_vmp(y, **kw, iterations=30)
    recovery_assertions(r, s_true, means, A)


# --------------------------------------------------------------------------- the kernel body on the host
def host_params(d, K, p0, mu0, V0, nu0, S0, m_init, Vm_init, nu_init, S_init, A_prior=None, A_init=None, A_known=None):
    """The fp64 constant block of rxg_hmm_gauss_vmp_f32 (rxg::hmmg::layout) from fp32-rounded inputs."""
    A = f32(A_known if A_known is not None else A_prior)
    Ai = f32(A_init) if A_known is None else np.zeros((K, K))
    blocks = []
    for k in range(K):
        V0k, S0k = f32(V0[k]), f32(S0[k])
        Vk = f32(Vm_init[k])
        blocks.append(np.concatenate([
            f32(mu0[k]), np.linalg.inv(V0k).ravel(), np.linalg.inv(V0k) @ f32(mu0[k]), [np.linalg.slogdet(V0k)[1]],
            np.linalg.inv(S0k).ravel(), [np.linalg.slogdet(S0k)[1]], [f32(nu0[k])], [multigammaln(0.5 * f32(nu0[k]), d)],
            f32(m_init[k]), (0.5 * (Vk + Vk.T)).ravel(), [f32(nu_init[k])], np.linalg.inv(f32(S_init[k])).ravel()]))
    return np.concatenate([f32(p0), A.ravel(), Ai.ravel(), *blocks])


def _host_harness():
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    so = os.path.join(ROOT, "tests", "c", "_hmm_gauss_host.so")
    src = os.path.join(ROOT, "tests", "c", "hmm_gauss_host_harness.cu")
    hdrs = [os.path.join(ROOT, "rxinfer.jl_b200", "csrc", h) for h in ("rxg_hmm_gauss.cuh", "rxg_hmm.cuh")]
    if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(p) for p in [src, *hdrs]):
        subprocess.run([nvcc, "-O2", "-std=c++17", "-Wno-deprecated-gpu-targets", "-shared", "-Xcompiler", "-fPIC", "-o", so,
                        src], check=True)
    return ctypes.CDLL(so)


def run_host(lib, y, kw, iterations, prm=None):
    T, d, nb = y.shape
    K = len(kw["p0"])
    la = "A_prior" in kw
    prm = host_params(d, K, **kw) if prm is None else prm
    z = lambda *s: np.zeros(s, np.float32)
    its = iterations
    out = dict(s_prob=z(T, K, nb), s0_prob=z(K, nb), A_alpha=z(K, K, nb), m_mean=z(K, d, nb), m_cov=z(K, d, d, nb),
               w_df=z(K, nb), w_inv_scale=z(K, d, d, nb), free_energy=np.zeros((its, nb)), hist_s=z(its, T, K, nb),
               hist_A=z(its, K, K, nb), hist_m_mean=z(its, K, d, nb), hist_m_cov=z(its, K, d, d, nb), hist_w_df=z(its, K, nb),
               hist_w_inv_scale=z(its, K, d, d, nb), status=np.zeros(nb, np.int32))
    P = lambda a: a.ctypes.data_as(ctypes.c_void_p)
    yy = np.ascontiguousarray(y, np.float32)
    names = ("s_prob", "s0_prob", "A_alpha", "m_mean", "m_cov", "w_df", "w_inv_scale", "free_energy", "hist_s", "hist_A",
             "hist_m_mean", "hist_m_cov", "hist_w_df", "hist_w_inv_scale", "status")
    rc = lib.hmm_gauss_host_run(d, K, T, ctypes.c_longlong(nb), its, int(la), P(np.ascontiguousarray(prm, np.float64)), P(yy),
                                *(P(out[k]) for k in names))
    assert rc == 0
    if not la:
        out["A_alpha"] = out["hist_A"] = None
    return out


def per_chain_rel(got, want):
    ax = tuple(range(got.ndim - 1))
    return (np.sqrt(((got - want) ** 2).sum(ax)) / np.maximum(np.sqrt((want ** 2).sum(ax)), 1e-30)).max()


def gate(case, r, ref, chains=None, tol_mean=1e-5, tol_cov=1e-4, tol_s=1e-3, fe_tol=1e-5, hist=3.0):
    """Per chain: E[m], alpha_A, nu at tol_mean relative L2; cov m, W inverse scale at tol_cov; q(s_t), q(s_0) at tol_s
    absolute; the KeepEach histories at ``hist`` times those; the free energy at fe_tol relative to max(|F|, 1) and
    non-increasing.  Returns the worst error per output."""
    sel = (lambda v: v[..., chains]) if chains is not None else (lambda v: v)
    assert np.all(sel(np.asarray(r["status"])) == 0), case
    worst = {}
    gates = dict(A_alpha=tol_mean, m_mean=tol_mean, w_df=tol_mean, m_cov=tol_cov, w_inv_scale=tol_cov)
    for k, tol in gates.items():
        for key, t in ((k, tol), ("hist_" + k.replace("A_alpha", "A"), hist * tol)):
            if ref.get(key) is None or r.get(key) is None:
                continue
            e = per_chain_rel(sel(np.asarray(r[key], np.float64)), sel(ref[key]))
            worst[key] = e
            assert e < t, f"{case}: {key} {e:.3g}"
    for k, t in (("s_prob", tol_s), ("s0_prob", tol_s), ("hist_s", hist * tol_s)):
        if r.get(k) is None:
            continue
        e = np.abs(sel(np.asarray(r[k], np.float64)) - sel(ref[k])).max()
        worst[k] = e
        assert e < t, f"{case}: {k} {e:.3g}"
    fe, fr = sel(np.asarray(r["free_energy"])), sel(ref["free_energy"])
    e = (np.abs(fe - fr) / np.maximum(np.abs(fr), 1.0)).max()
    worst["free_energy"] = e
    assert e < fe_tol, f"{case}: free energy {e:.3g}"
    assert np.all(np.diff(fe, axis=0) <= 2 * fe_tol * np.maximum(np.abs(fe[:-1]), 1.0)), case
    return worst


@pytest.mark.parametrize("d", [1, 2, 3, 4])
def test_kernel_body_on_the_host_matches_the_reference(d):
    lib = _host_harness()
    for K in (2, 3, 5, 8):
        for T in (1, 7, 300):
            for la in (True, False):
                y, kw = random_problem(d, K, T, 3, seed=1000 * d + 10 * K + T + la, learn_A=la, p_missing=0.15)
                for its in (1, 20):
                    r = run_host(lib, y, kw, its)
                    gate(f"d={d} K={K} T={T} its={its} learn A={la}", r, reference_on_f32(y, kw, its), tol_s=1e-3)


def test_kernel_body_on_the_host_flags_bad_chains_only():
    """A non-finite datum that is not an all-NaN step flags its chain BAD_ARG and the step is read as missing; a datum that
    makes every emission weight vanish flags NAN; a non-SPD inverse scale flags NOT_SPD; the neighbours keep their results."""
    lib = _host_harness()
    y, kw = random_problem(2, 3, 30, 4, seed=9, p_missing=0.1)
    y[5, 0, 1] = np.inf
    y[8, 1, 3] = np.nan                                                  # one component only: not a missing step
    y[3, :, 2] = 3e38
    r = run_host(lib, y, kw, 3)
    assert list(r["status"]) == [0, 1, 5, 1]
    ym = y.copy()
    ym[5, :, 1] = np.nan
    ym[8, :, 3] = np.nan
    ym[:, :, 2] = np.nan                                                 # (chain 2 is not compared)
    ref = reference_on_f32(ym, kw, 3)
    gate("flagged neighbours", r, ref, chains=[0], tol_s=1e-3)
    for b in (1, 3):                                                     # read as missing: same results as the missing step
        sub = {k: (v[..., [b]] if v is not None and k not in ("free_energy",) else v) for k, v in r.items()}
        sub["status"] = np.zeros(1, np.int32)
        sub["free_energy"] = r["free_energy"][:, [b]]
        gate(f"chain {b}", sub, {k: (v[..., [b]] if isinstance(v, np.ndarray) and v.ndim and v.shape[-1] == 4 else v)
                                  for k, v in ref.items()}, tol_s=1e-3)
    prm = host_params(2, 3, **{k: f32(v) for k, v in kw.items()})
    blk = 3 * 2 + 4 * 4 + 5
    bad = prm.copy()
    bad[3 + 2 * 9 + blk + (3 * 2 + 3 * 4 + 5):][:4] = [1.0, 2.0, 2.0, 1.0]   # inv(S_init) of state 1: indefinite
    r = run_host(lib, y[..., [0]], kw, 2, prm=bad)
    assert list(r["status"]) == [4]


# --------------------------------------------------------------------------- host-side argument handling
def test_model_arrays_and_the_univariate_spelling(rx):
    from rxinfer_jl_b200 import (DirichletCollection, GammaShapeRate, MvNormalMeanCovariance, NormalMeanVariance, PointMass,
                                 Wishart, vague)
    from rxinfer_jl_b200.inference import gaussian_hidden_markov_model, gaussian_hmm_arguments
    y, kw = random_problem(1, 2, 50, 3, seed=5)
    mv = gaussian_hidden_markov_model(p0=kw["p0"], A=DirichletCollection(kw["A_prior"]),
                                      m_prior=[MvNormalMeanCovariance(kw["mu0"][k], kw["V0"][k]) for k in range(2)],
                                      w_prior=[Wishart(kw["nu0"][k], kw["S0"][k]) for k in range(2)])
    init_mv = {"A": DirichletCollection(kw["A_init"]), "m": [MvNormalMeanCovariance(kw["m_init"][k], kw["Vm_init"][k])
                                                              for k in range(2)],
               "w": [Wishart(kw["nu_init"][k], kw["S_init"][k]) for k in range(2)]}
    uv = gaussian_hidden_markov_model(p0=kw["p0"], A=DirichletCollection(kw["A_prior"]),
                                      m_prior=[NormalMeanVariance(kw["mu0"][k, 0], kw["V0"][k, 0, 0]) for k in range(2)],
                                      w_prior=[GammaShapeRate(kw["nu0"][k] / 2, 1 / (2 * kw["S0"][k, 0, 0])) for k in range(2)])
    init_uv = {"A": DirichletCollection(kw["A_init"]), "m": [NormalMeanVariance(kw["m_init"][k, 0], kw["Vm_init"][k, 0, 0])
                                                              for k in range(2)],
               "w": [GammaShapeRate(kw["nu_init"][k] / 2, 1 / (2 * kw["S_init"][k, 0, 0])) for k in range(2)]}
    a_mv, a_uv = gaussian_hmm_arguments(mv, init_mv), gaussian_hmm_arguments(uv, init_uv)
    r_mv = hmm_gauss_vmp(y, **a_mv, iterations=6)
    r_uv = hmm_gauss_vmp(y, **a_uv, iterations=6)
    for k in ("s_prob", "A_alpha", "m_mean", "m_cov", "w_df", "w_inv_scale", "free_energy"):
        assert np.abs(r_mv[k] - r_uv[k]).max() < 1e-9 * max(1.0, np.abs(r_mv[k]).max()), k
    assert np.abs(r_mv["free_energy"] - hmm_gauss_vmp(y, **kw, iterations=6)["free_energy"]).max() < 1e-9 * 1e3
    # a known A, and the refusals of the argument conversion
    known = gaussian_hidden_markov_model(p0=kw["p0"], A=PointMass(np.eye(2) * 0.8 + 0.1), m_prior=mv.m_prior,
                                         w_prior=mv.w_prior)
    args = gaussian_hmm_arguments(known, {"m": init_mv["m"], "w": init_mv["w"], "s": vague(DirichletCollection, (2, 2))})
    assert "A_known" in args and "A_prior" not in args
    with pytest.raises(ValueError, match="initialization"):
        gaussian_hmm_arguments(mv, {"m": init_mv["m"], "w": init_mv["w"]})                 # learned A without q(A)
    with pytest.raises(ValueError, match="initialization"):
        gaussian_hmm_arguments(mv, {"A": init_mv["A"], "w": init_mv["w"]})
    with pytest.raises(ValueError, match="2 marginals for K = 3|K = 3"):
        gaussian_hmm_arguments(gaussian_hidden_markov_model(p0=np.full(3, 1 / 3), A=DirichletCollection(np.ones((3, 3))),
                                                            m_prior=mv.m_prior, w_prior=mv.w_prior),
                               dict(init_mv, A=DirichletCollection(np.ones((3, 3)))))
    with pytest.raises(TypeError, match="DirichletCollection or PointMass"):
        gaussian_hmm_arguments(gaussian_hidden_markov_model(p0=kw["p0"], A=np.eye(2), m_prior=mv.m_prior,
                                                            w_prior=mv.w_prior), init_mv)


def test_infer_refusals_before_the_device(rx):
    """infer refuses other factorisations, predictvars, datastream and bad data before it needs a device (context=object()
    would fail on any use), so these run with and without a GPU."""
    import torch
    from rxinfer_jl_b200 import (DirichletCollection, GaussianHMMConstraints, HMMConstraints, KeepEach, KeepLast, MeanField,
                                 MvNormalMeanCovariance, Wishart, gaussian_hidden_markov_model)
    y, kw = random_problem(2, 3, 20, 2, seed=3)
    model = gaussian_hidden_markov_model(p0=kw["p0"], A=DirichletCollection(kw["A_prior"]),
                                         m_prior=[MvNormalMeanCovariance(kw["mu0"][k], kw["V0"][k]) for k in range(3)],
                                         w_prior=[Wishart(kw["nu0"][k], kw["S0"][k]) for k in range(3)])
    init = {"A": DirichletCollection(kw["A_init"]), "m": [MvNormalMeanCovariance(kw["m_init"][k], kw["Vm_init"][k])
                                                           for k in range(3)],
            "w": [Wishart(kw["nu_init"][k], kw["S_init"][k]) for k in range(3)]}
    data = {"y": torch.as_tensor(y, dtype=torch.float32)}
    call = lambda **k: rx.infer(**{**dict(model=model, data=data, constraints=GaussianHMMConstraints(),
                                          initialization=init, iterations=2, context=object()), **k})
    for c in (MeanField(), HMMConstraints(), None, "q(s)q(A)q(m)q(w)"):
        with pytest.raises(ValueError, match=r"q\(s_0, s\) q\(A\)"):
            call(constraints=c)
    with pytest.raises(NotImplementedError, match="predictvars"):
        call(predictvars={"y": KeepLast()})
    with pytest.raises(NotImplementedError, match="datastream"):
        call(data=None, datastream=iter([]))
    with pytest.raises(KeyError, match="'y'"):
        call(data={"x": data["y"]})
    with pytest.raises(ValueError, match=r"d = 2, batch\] .*got \(20, 3, 2\)"):
        call(data={"y": torch.zeros(20, 3, 2)})
    with pytest.raises(NotImplementedError, match="s_0"):
        call(returnvars={"s_0": KeepEach()})
    with pytest.raises(NotImplementedError, match="returnvars"):
        call(returnvars={"x": KeepLast()})
    with pytest.raises(ValueError, match="initialization"):
        call(initialization={"m": init["m"], "w": init["w"]})
    assert GaussianHMMConstraints() == GaussianHMMConstraints() and GaussianHMMConstraints() != HMMConstraints()
    if not torch.cuda.is_available():
        with pytest.raises(Exception):           # and needs a device otherwise (no CPU fallback)
            rx.infer(model=model, data=data, constraints=GaussianHMMConstraints(), initialization=init, iterations=2)
