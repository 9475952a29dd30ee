"""fp64 reference of the Delta node (z := f(x) with Linearization() / Unscented()) on Gaussian chains: the EKF / ERTS
and UKF / URTS smoother, the streaming filter, the per-datum VMP of the paper's pendulum (paper/example.jl) and its
``dataset``.  Functions are Python callables on 1-D arrays; Linearization takes their analytic Jacobians.

Time convention as ``oracle.lgssm``: x[1] ~ N(m0, S0), x[t] = f(x[t-1]) + N(0, P), y[t] ~ N(B x[t] or g(x[t]), Q),
arrays y[T, m, batch] and outputs mean[T, d, batch], cov[T, d, d, batch]."""
from __future__ import annotations

import numpy as np

from .julia_rng import StableRNG

UT_DEFAULTS = (1e-3, 2.0, 0.0)     # ReactiveMP's Unscented(alpha, beta, kappa) defaults


class Fn:
    """A map h: R^n -> R^k with its Jacobian (only Linearization uses it)."""

    def __init__(self, h, jac):
        self.h, self.jac = h, jac


def linear(A):
    A = np.asarray(A, np.float64)
    return Fn(lambda x: A @ x, lambda x: A)


def moments(fn, mu, S, method, ut=UT_DEFAULTS):
    """(mz, Szz, Sxz) of z = h(x), x ~ N(mu, S)."""
    mu, S = np.asarray(mu, np.float64), np.asarray(S, np.float64)
    if method == "linearization":
        J = np.atleast_2d(fn.jac(mu))
        return np.asarray(fn.h(mu), np.float64), J @ S @ J.T, S @ J.T
    alpha, beta, kappa = ut
    n = mu.shape[0]
    lam = alpha ** 2 * (n + kappa) - n
    L = np.linalg.cholesky((n + lam) * S)
    X = [mu] + [mu + L[:, i] for i in range(n)] + [mu - L[:, i] for i in range(n)]
    Z = np.array([np.asarray(fn.h(x), np.float64) for x in X])
    wm = np.full(2 * n + 1, 0.5 / (n + lam))
    wc = wm.copy()
    wm[0] = lam / (n + lam)
    wc[0] = wm[0] + 1.0 - alpha ** 2 + beta
    mz = wm @ Z
    dZ, dX = Z - mz, np.array(X) - mu
    return mz, (wc[:, None] * dZ).T @ dZ, (wc[:, None] * dX).T @ dZ


def _update(m, S, y, g, B, Q, method, ut):
    if g is None:
        my, Syy, Sxy = B @ m, B @ S @ B.T, S @ B.T
    else:
        my, Syy, Sxy = moments(g, m, S, method, ut)
    K = Sxy @ np.linalg.inv(Syy + Q)
    S = S - K @ (Syy + Q) @ K.T
    return m + K @ (y - my), 0.5 * (S + S.T)


def _predict(m, S, f, P, method, ut):
    mz, Szz, Sxz = moments(f, m, S, method, ut)
    return mz, Szz + P, Sxz


def smooth_chain(y, f, P, m0, S0, method, g=None, B=None, Q=None, mask=None, ut=UT_DEFAULTS):
    """One chain: y[T, m] -> (smoothed mean [T, d], cov [T, d, d], filtered mean, cov)."""
    T, d = y.shape[0], len(m0)
    fm, fc = np.zeros((T, d)), np.zeros((T, d, d))
    m, S = np.asarray(m0, np.float64), np.asarray(S0, np.float64)
    for t in range(T):
        if t > 0:
            m, S, _ = _predict(m, S, f, P, method, ut)
        if mask is None or mask[t]:
            m, S = _update(m, S, y[t], g, B, Q, method, ut)
        fm[t], fc[t] = m, S
    sm, sc = fm.copy(), fc.copy()
    for t in range(T - 2, -1, -1):
        mp, Sp, Sxz = _predict(fm[t], fc[t], f, P, method, ut)
        G = Sxz @ np.linalg.inv(Sp)
        sm[t] = fm[t] + G @ (sm[t + 1] - mp)
        sc[t] = fc[t] + G @ (sc[t + 1] - Sp) @ G.T
    return sm, sc, fm, fc


def smooth(y, f, P, m0, S0, method, g=None, B=None, Q=None, mask=None, ut=UT_DEFAULTS):
    """Batched: y[T, m, batch], mask[T, batch] or None -> dict of mean / cov (smoothed) and filt_mean / filt_cov."""
    T, _, nb = y.shape
    d = len(m0)
    out = {k: np.zeros((T, d, nb)) for k in ("mean", "filt_mean")}
    out.update({k: np.zeros((T, d, d, nb)) for k in ("cov", "filt_cov")})
    for b in range(nb):
        r = smooth_chain(y[:, :, b], f, P, m0, S0, method, g, B, Q, None if mask is None else mask[:, b], ut)
        for k, v in zip(("mean", "cov", "filt_mean", "filt_cov"), r):
            out[k][..., b] = v
    return out


def filter_stream(y, f, P, m, S, method, g=None, B=None, Q=None, mask=None, ut=UT_DEFAULTS):
    """Streaming filter of one chain from the carry N(m, S): every datum predicts through f first."""
    T, d = y.shape[0], len(m)
    fm, fc = np.zeros((T, d)), np.zeros((T, d, d))
    for t in range(T):
        m, S, _ = _predict(m, S, f, P, method, ut)
        if mask is None or mask[t]:
            m, S = _update(m, S, y[t], g, B, Q, method, ut)
        fm[t], fc[t] = m, S
    return fm, fc


def vmp_gamma_stream(y, f, P, c, m, S, shape, rate, iters, method, mask=None, ut=UT_DEFAULTS):
    """The pendulum's per-datum VMP for one chain (paper/example.jl): the message through f from the autoupdated prior
    N(m, S) (plus P), then `iters` times q(x) ∝ m_f(x) N(y | c'x, 1/E[tau]) and
    q(tau) = Gamma(shape0 + 1/2, rate0 + E_q[(y - c'x)^2] / 2); the carry q(x), q(tau) is the next datum's prior (and
    its initial q(tau)).  Returns mean [T, d], cov [T, d, d], shape [T], rate [T]."""
    c = np.asarray(c, np.float64)
    T, d = len(y), len(m)
    om, oc, oa, ob = np.zeros((T, d)), np.zeros((T, d, d)), np.zeros(T), np.zeros(T)
    for t in range(T):
        mp, Sp, _ = _predict(m, S, f, P, method, ut)
        a0, b0 = shape, rate
        m, S = mp, Sp
        if mask is None or mask[t]:
            for _ in range(iters):
                s = c @ Sp @ c + rate / shape
                k = Sp @ c / s
                m, S = mp + k * (y[t] - c @ mp), Sp - np.outer(k, k) * s
                shape, rate = a0 + 0.5, b0 + 0.5 * ((y[t] - c @ m) ** 2 + c @ S @ c)
        om[t], oc[t], oa[t], ob[t] = m, S, shape, rate
    return om, oc, oa, ob


# ------------------------------------------------------------------ the paper's pendulum (paper/example.jl)
DT, GRAV = 0.01, 9.81
PENDULUM = Fn(lambda x: np.array([x[0] + x[1] * DT, x[1] - GRAV * np.sin(x[0]) * DT]),
              lambda x: np.array([[1.0, DT], [-GRAV * np.cos(x[0]) * DT, 1.0]]))
PENDULUM_INIT = dict(mean=np.array([0.5, 0.0]), cov=0.01 * np.eye(2), shape=1.0, scale=100.0)


def dataset(T, precision=1.0, seed=42):
    """``dataset(; T, precision, seed)`` of paper/example.jl: noiseless pendulum states and observations of the angle
    with precision ``precision``, drawn with StableRNG(seed).  observations[1] is never assigned there and stays 0."""
    rng = StableRNG(seed)
    states = np.zeros((2, T))
    obs = np.zeros(T)
    states[:, 0] = [0.5, 0.0]
    for t in range(1, T):
        states[:, t] = PENDULUM.h(states[:, t - 1])
        obs[t] = states[0, t] + rng.randn() / np.sqrt(precision)     # rand(rng, NormalMeanPrecision(x, precision))
    return np.arange(1, T + 1) * DT, states, obs
