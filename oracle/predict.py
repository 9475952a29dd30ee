"""fp64 oracle for the predictive distributions of the observations (``result.predictions``).

TEST INFRASTRUCTURE ONLY (see oracle/__init__.py).
"""
from __future__ import annotations

import numpy as np

from . import rules as R
from .lgssm import _bc, _pack, smooth_reference_schedule


def predict_reference_schedule(y, A, B, P, Q, m0, S0, mask=None, u=None, transition_first=False, horizon=0):
    """Predictions of the observations as the reference computes them (``result.predictions``,
    /root/reference/src/inference/batch.jl:203-246): the message toward ``y[t]``.

    ``y`` is padded with ``horizon`` missing steps (the forecast graph of ``model_1``,
    test/inference/prediction_tests.jl:197-213) and run through ``smooth_reference_schedule``.  Per step the
    cavity ``prod(fwd_t, bwd_t)`` (every message into x[t] except the one from y[t]) is formed in (xi, W), converted,
    and pushed through ``*(:out)`` with B and ``MvNormalMeanCovariance(:out)`` with Q.  This is deliberately not the
    closed form the kernels use, so that the two check each other.

    ``mask``: [T, batch] per chain, [T] shared, or None.  Returns dict(pred_mean[T+H, m, batch],
    pred_cov[T+H, m, m, batch], mean / cov (posteriors of x[1..T]), fc_mean[H, d, batch], fc_cov[H, d, d, batch]).
    """
    y = np.asarray(y, dtype=np.float64)
    T, m, batch = y.shape
    H = int(horizon)
    mk = np.ones((T, batch), dtype=bool) if mask is None else np.asarray(mask).astype(bool)
    if mk.ndim == 1:
        mk = np.broadcast_to(mk[:, None], (T, batch))
    yp = np.concatenate([y, np.zeros((H, m, batch))], axis=0)
    mkp = np.concatenate([mk, np.zeros((H, batch), dtype=bool)], axis=0)
    r = smooth_reference_schedule(yp, A, B, P, Q, m0, S0, mkp, return_messages=True, u=u,
                                  transition_first=transition_first)
    d = np.asarray(A).shape[-1]
    Bb = _bc(B, batch, (m, d)); Qb = _bc(Q, batch, (m, m))
    pm = np.zeros((T + H, batch, m)); pS = np.zeros((T + H, batch, m, m))
    for t in range(T + H):
        xi, W = R.prod_gaussian_wmp(R.meancov_to_wmp(r["fwd_mean"][t], r["fwd_cov"][t]), (r["bwd_xi"][t], r["bwd_W"][t]))
        cavity = R.wmp_to_meancov(xi, W)
        pm[t], pS[t] = R.mvnormal_meancov_out(R.multiplication_out(Bb, cavity), Qb)
    pred_mean, pred_cov = _pack(pm, pS)
    return dict(pred_mean=pred_mean, pred_cov=pred_cov, mean=r["mean"][:T], cov=r["cov"][:T],
                fc_mean=r["mean"][T:], fc_cov=r["cov"][T:])


def predict_closed_form(y, A, B, P, Q, m0, S0, mask=None, u=None, transition_first=False, horizon=0):
    """The closed form the kernels evaluate, over Kalman + RTS (kalman_rts): with D_t = Q - B S_s B',
    observed y[t] -> N(y - Q D^-1 (y - B mu_s), Q D^-1 Q); missing -> N(B mu_s, B S_s B' + Q); forecasts step
    (x, S) <- (A x + u, A S A' + P) from the last smoothed state.  Same layouts as predict_reference_schedule."""
    from .lgssm import kalman_rts
    y = np.asarray(y, dtype=np.float64)
    T, m, batch = y.shape
    d = np.asarray(A).shape[-1]
    H = int(horizon)
    mk = np.ones((T, batch), dtype=bool) if mask is None else np.asarray(mask).astype(bool)
    if mk.ndim == 1:
        mk = np.broadcast_to(mk[:, None], (T, batch))
    r = kalman_rts(y, A, B, P, Q, m0, S0, mk, u=u, transition_first=transition_first)
    Ab = _bc(A, batch, (d, d)); Bb = _bc(B, batch, (m, d)); Pb = _bc(P, batch, (d, d)); Qb = _bc(Q, batch, (m, m))
    ub = _bc(np.zeros(d) if u is None else u, batch, (d,))
    mu = np.transpose(r["mean"], (0, 2, 1)); S = np.transpose(r["cov"], (0, 3, 1, 2))       # [T, batch, d(, d)]
    yb = np.transpose(y, (0, 2, 1))
    Bt = np.swapaxes(Bb, -1, -2); At = np.swapaxes(Ab, -1, -2)
    pm = np.zeros((T + H, batch, m)); pS = np.zeros((T + H, batch, m, m))
    for t in range(T):
        BSB = Bb @ S[t] @ Bt
        Dt = Qb - BSB
        X = np.linalg.solve(Dt, Qb)                                          # D^-1 Q, K = Q D^-1 = X'
        obs_mean = yb[t] - R.mv(np.swapaxes(X, -1, -2), yb[t] - R.mv(Bb, mu[t]))
        pm[t] = np.where(mk[t][:, None], obs_mean, R.mv(Bb, mu[t]))
        pS[t] = np.where(mk[t][:, None, None], Qb @ X, BSB + Qb)
    x, Sx = mu[T - 1], S[T - 1]
    fm = np.zeros((H, batch, d)); fS = np.zeros((H, batch, d, d))
    for k in range(H):
        x, Sx = R.mv(Ab, x) + ub, Ab @ Sx @ At + Pb
        fm[k], fS[k] = x, Sx
        pm[T + k], pS[T + k] = R.mv(Bb, x), Bb @ Sx @ Bt + Qb
    pred_mean, pred_cov = _pack(pm, pS)
    fc_mean, fc_cov = _pack(fm, fS)
    return dict(pred_mean=pred_mean, pred_cov=pred_cov, mean=r["mean"], cov=r["cov"], fc_mean=fc_mean, fc_cov=fc_cov)
