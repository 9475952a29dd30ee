"""fp64 reference of the VMP that learns the transition matrix per chain (rxg_lgssm_vmp_transition_f32: RxInfer's
ContinuousTransition with a linear reshape), and its CPU checks.

Model (per chain): a = vec(A) (row-major, a[i d + j] = A[i, j]) ~ N(ma0, Va0); w_p ~ Wishart(nu_p0, inv(Psi_p0)) (else P
known); w_q likewise (else Q known); x[1] ~ N(m0, S0) (or one transition earlier); x[t] ~ N(A x[t-1] + u, inv(w_p));
y[t] ~ N(B x[t], inv(w_q)); q(x) q(a) q(w_p) q(w_q).  ``lgssm_continuous_transition`` runs one iteration as
  q(x)   a standard Kalman filter + RTS smoother at (E[A], inv(E[w_p]), inv(E[w_q])) per chain in which the factor
         exp(-1/2 x' Xi x), Xi = E[(A - E[A])' E[w_p] (A - E[A])] = L L', on the source state of every transition is a zero
         pseudo-observation through L' with identity noise;
  q(a)   Lambda = Va0^-1 + E[w_p] (x) Sxx, xi = Va0^-1 ma0 + vec(E[w_p] M) from the smoothed pair statistics
         Sxx = sum E[x_t x_t'], M = sum E[(x_{t+1} - u) x_t'];
  q(w_p) with R_p = sum E_{q(x) q(a)}[(x_{t+1} - A x_t - u)(...)'] at the new q(a) (pair covariances, no large moments);
  q(w_q) as test_vmp_noise;
  F      in closed form (the tilted evidence + 1/2 tr(Wbar_p (R_p,new - R_p,old)) + KL(q(a) || prior) + the Wishart
         blocks) and, with ``definition=True``, from its definition with a dense Gaussian q(x) over every latent state.
"""
import numpy as np
import pytest
import torch

from test_vmp_noise import _Ew_terms, _wishart_block, lgssm_wishart_noise
from test_vmp_wishart import _mvdigamma, random_problem, wishart_kl

MODES = ["A", "AP", "AQ", "APQ"]


def _kron_contract(Sa, S, d):
    """K[i, l] = sum_{j,k} Sa[(i,j),(l,k)] S[j, k], batched."""
    return np.einsum("bijlk,bjk->bil", Sa.reshape(-1, d, d, d, d), S)


def _xi(Sa, W, d):
    """Xi[j, k] = sum_{i,l} W[i, l] Sa[(i,j),(l,k)], batched."""
    return np.einsum("bil,bijlk->bjk", W, Sa.reshape(-1, d, d, d, d))


def _pseudo_update(mu, S, H, R, z, on):
    """Kalman update of (mu, S) with observation z = H x + N(0, R) where ``on``; returns the -log evidence increment."""
    Sinn = H @ S @ np.swapaxes(H, -1, -2) + R
    Si = np.linalg.inv(Sinn)
    e = z - np.einsum("bij,bj->bi", H, mu)
    K = S @ np.swapaxes(H, -1, -2) @ Si
    mu_n = mu + np.einsum("bij,bj->bi", K, e)
    S_n = S - K @ Sinn @ np.swapaxes(K, -1, -2)
    S_n = 0.5 * (S_n + np.swapaxes(S_n, -1, -2))
    nle = 0.5 * (np.einsum("bi,bij,bj->b", e, Si, e) + np.linalg.slogdet(Sinn)[1])
    o = on[:, None]
    return np.where(o, mu_n, mu), np.where(o[..., None], S_n, S), np.where(on, nle, 0.0)


def tilted_smoother(yb, mk, A, Pb, Qb, B, m0, S0, u, tf, Lx):
    """Per-chain Kalman filter + RTS smoother (fp64) with the tilt through Lx on every source state.  yb[T, batch, m];
    A, Pb, Lx [batch, d, d]; Qb [batch, m, m].  Returns the smoothed means / covariances of the source states and of
    every state ([n, batch, ...], x_0 first with tf), the cross covariances cov(x_{t+1}, x_t) [n - 1, batch, d, d],
    the filter's -log evidence and the last-step smoothed state (= filtered)."""
    T, batch, m = yb.shape
    d = A.shape[-1]
    I = np.broadcast_to(np.eye(d), (batch, d, d))
    Lt = np.swapaxes(Lx, -1, -2)
    zero = np.zeros((batch, d))
    allon = np.ones(batch, bool)
    mu = np.broadcast_to(m0, (batch, d)).copy(); S = np.broadcast_to(S0, (batch, d, d)).copy()
    Bb = np.broadcast_to(B, (batch, m, d))
    nle = np.zeros(batch)
    fm, fS = [], []                                         # filtered (tilted) states that start a transition
    for t in range(T):
        if t > 0 or tf:
            if t == 0:
                mu, S, inc = _pseudo_update(mu, S, Lt, I, zero, allon)
                nle += inc
                fm.append(mu); fS.append(S)
            mu = np.einsum("bij,bj->bi", A, mu) + u
            S = A @ S @ np.swapaxes(A, -1, -2) + Pb
            S = 0.5 * (S + np.swapaxes(S, -1, -2))
        mu, S, inc = _pseudo_update(mu, S, Bb, Qb, yb[t], mk[t])
        nle += inc + np.where(mk[t], 0.5 * m * np.log(2 * np.pi), 0.0)
        if t < T - 1:
            mu, S, inc = _pseudo_update(mu, S, Lt, I, zero, allon)
            nle += inc
            fm.append(mu); fS.append(S)
    n = len(fm) + 1
    sm, sS, cross = [None] * n, [None] * n, [None] * (n - 1)
    sm[-1], sS[-1] = mu, S
    for k in range(n - 2, -1, -1):
        Sp = A @ fS[k] @ np.swapaxes(A, -1, -2) + Pb
        G = fS[k] @ np.swapaxes(A, -1, -2) @ np.linalg.inv(Sp)
        sm[k] = fm[k] + np.einsum("bij,bj->bi", G, sm[k + 1] - np.einsum("bij,bj->bi", A, fm[k]) - u)
        sS[k] = fS[k] + G @ (sS[k + 1] - Sp) @ np.swapaxes(G, -1, -2)
        sS[k] = 0.5 * (sS[k] + np.swapaxes(sS[k], -1, -2))
        cross[k] = sS[k + 1] @ np.swapaxes(G, -1, -2)
    return dict(mean=np.stack(sm), cov=np.stack(sS), cross=np.stack(cross) if n > 1 else np.zeros((0, batch, d, d)),
                nle=nle, fmean=fm, fcov=fS)


def pair_stats(sm, sS, cross, u):
    """Sxx = sum_src (S_t + m_t m_t'), M = sum (cov(x_{t+1}, x_t) + (m_{t+1} - u) m_t')."""
    src_m, src_S = sm[:-1], sS[:-1]
    Sxx = (src_S + np.einsum("tbi,tbj->tbij", src_m, src_m)).sum(0)
    M = (cross + np.einsum("tbi,tbj->tbij", sm[1:] - u, src_m)).sum(0)
    return Sxx, M


def residual_R(sm, sS, cross, Abar, u):
    """sum_t E[(x_{t+1} - Abar x_t - u)(...)'] under the smoothed pairs, from pair covariances (no large moments)."""
    At = np.swapaxes(Abar, -1, -2)
    R = 0.0
    for t in range(sm.shape[0] - 1):
        C = cross[t]                                        # cov(x_{t+1}, x_t)
        V = sS[t + 1] - C @ At - Abar @ np.swapaxes(C, -1, -2) + Abar @ sS[t] @ At
        e = sm[t + 1] - np.einsum("bij,bj->bi", Abar, sm[t]) - u
        R = R + V + np.einsum("bi,bj->bij", e, e)
    return R


def kl_gauss(am, Sa, ma0, Va0):
    n = am.shape[-1]
    Vi = np.linalg.inv(Va0)
    dm = am - ma0
    return 0.5 * (np.einsum("ij,bji->b", Vi, Sa) + np.einsum("bi,ij,bj->b", dm, Vi, dm) - n
                  + np.linalg.slogdet(Va0)[1] - np.linalg.slogdet(Sa)[1])


def _dense_chain(yc, mkc, A, Wp, Wq, Xi, B, m0, S0, u, tf):
    """Dense Gaussian q(x) of one chain (x_0 included with tf): prior, transitions at (A, Wp), the tilt Xi on every
    source state and the observations at Wq.  Returns (mu [n, d], Sig [n d, n d])."""
    T, m = yc.shape
    d = A.shape[0]
    n = T + (1 if tf else 0)
    o = 1 if tf else 0
    J = np.zeros((n * d, n * d)); h = np.zeros(n * d)
    S0i = np.linalg.inv(S0)
    J[:d, :d] += S0i; h[:d] += S0i @ m0
    for t in range(1, n):
        a, b = slice((t - 1) * d, t * d), slice(t * d, (t + 1) * d)
        J[b, b] += Wp; J[a, a] += A.T @ Wp @ A + Xi
        J[b, a] -= Wp @ A; J[a, b] -= A.T @ Wp
        h[b] += Wp @ u; h[a] -= A.T @ Wp @ u
    for t in range(T):
        if mkc[t]:
            s = slice((t + o) * d, (t + o + 1) * d)
            J[s, s] += B.T @ Wq @ B
            h[s] += B.T @ Wq @ yc[t]
    Sig = np.linalg.inv(J)
    return (Sig @ h).reshape(n, d), Sig


def lgssm_continuous_transition(y, B, m0, S0, iterations, *, a_prior, a_init, P=None, Q=None, p_prior=None, p_init=None,
                                q_prior=None, q_init=None, mask=None, u=None, transition_first=False, definition=False,
                                stats_check=False):
    """y[T, m, batch]; mask None, [T, batch] or a shared [T] pattern; a_prior / a_init = (mean [d, d] or [d * d],
    covariance [d * d, d * d]) row-major.  Returns dict(mean[T, d, batch], cov[T, d, d, batch] of the last iteration;
    a_mean[iterations, d, d, batch], a_cov[iterations, n, n, batch]; df_p / inv_scale_p / E_Wp and df_q / inv_scale_q /
    E_Wq per iteration for the learned noises; free_energy[iterations, batch] (closed form) and, with ``definition``,
    free_energy_definition; with ``stats_check``, per iteration the pair-statistics and dense-joint Lambda, xi, R_p and
    the kernel's update form of R_p)."""
    y = np.asarray(y, dtype=np.float64)
    T, m, batch = y.shape
    B = np.asarray(B, np.float64)
    d = B.shape[1]
    n = d * d
    m0, S0 = np.asarray(m0, np.float64), np.asarray(S0, np.float64)
    uu = np.zeros(d) if u is None else np.asarray(u, np.float64)
    tf = bool(transition_first)
    mk = np.ones((T, batch), dtype=bool) if mask is None else np.asarray(mask).astype(bool)
    if mk.ndim == 1:
        mk = np.broadcast_to(mk[:, None], (T, batch)).copy()
    ma0 = np.asarray(a_prior[0], np.float64).reshape(n); Va0 = np.asarray(a_prior[1], np.float64)
    Va0i = np.linalg.inv(Va0)
    am = np.broadcast_to(np.asarray(a_init[0], np.float64).reshape(n), (batch, n)).copy()
    Sa = np.broadcast_to(np.asarray(a_init[1], np.float64), (batch, n, n)).copy()
    lp, lq = P is None, Q is None
    Wp = (np.broadcast_to(np.asarray(p_init, np.float64), (batch, d, d)) if lp else
          np.broadcast_to(np.linalg.inv(np.asarray(P, np.float64)), (batch, d, d))).copy()
    Wq = (np.broadcast_to(np.asarray(q_init, np.float64), (batch, m, m)) if lq else
          np.broadcast_to(np.linalg.inv(np.asarray(Q, np.float64)), (batch, m, m))).copy()
    yb = np.transpose(y, (0, 2, 1))
    Np = T - 1 + int(tf)
    hist = {k: [] for k in ("a_mean", "a_cov", "df_p", "inv_scale_p", "E_Wp", "df_q", "inv_scale_q", "E_Wq",
                            "free_energy", "free_energy_definition", "stats")}
    for _ in range(iterations):
        Abar = am.reshape(batch, d, d)
        Pb = np.linalg.inv(Wp) if lp else np.broadcast_to(np.asarray(P, np.float64), (batch, d, d))
        Qb = np.linalg.inv(Wq) if lq else np.broadcast_to(np.asarray(Q, np.float64), (batch, m, m))
        Xi = _xi(Sa, Wp, d)
        Lx = np.linalg.cholesky(Xi)
        r = tilted_smoother(yb, mk, Abar, Pb, Qb, B, m0, S0, uu, tf, Lx)
        fe = r["nle"].copy()
        sm, sS, cross = r["mean"], r["cov"], r["cross"]
        # ---- q(a) with the Wbar_p of this sweep
        Sxx, M = pair_stats(sm, sS, cross, uu)
        Lam = Va0i[None] + np.einsum("bil,bjk->bijlk", Wp, Sxx).reshape(batch, n, n)
        xi = (Va0i @ ma0)[None] + (Wp @ M).reshape(batch, n)
        Sa_n = np.linalg.inv(Lam)
        Sa_n = 0.5 * (Sa_n + np.swapaxes(Sa_n, -1, -2))
        am_n = np.einsum("bij,bj->bi", Sa_n, xi)
        An = am_n.reshape(batch, d, d)
        K_old, K_new = _kron_contract(Sa, Sxx, d), _kron_contract(Sa_n, Sxx, d)
        R_old = residual_R(sm, sS, cross, Abar, uu) + K_old
        R_new = residual_R(sm, sS, cross, An, uu) + K_new
        fe += 0.5 * np.einsum("bij,bji->b", Wp, R_new - R_old) + kl_gauss(am_n, Sa_n, ma0, Va0)
        if stats_check:
            Dl = An - Abar
            Sxr = np.swapaxes(M, -1, -2) - Sxx @ np.swapaxes(Abar, -1, -2)          # sum E[x_t r_t'] at Abar_old
            R_upd = (residual_R(sm, sS, cross, Abar, uu) + Dl @ Sxx @ np.swapaxes(Dl, -1, -2) - Dl @ Sxr
                     - np.swapaxes(Sxr, -1, -2) @ np.swapaxes(Dl, -1, -2) + K_new)
            dense = {"Lam": [], "xi": [], "R_new": []}
            for c in range(batch):
                mu, Sig = _dense_chain(yb[:, c], mk[:, c], Abar[c], Wp[c], Wq[c], Xi[c], B, m0, S0, uu, tf)
                nst = mu.shape[0]
                blk = lambda s, t: Sig[s * d:(s + 1) * d, t * d:(t + 1) * d]
                Sxx_d = sum(blk(t, t) + np.outer(mu[t], mu[t]) for t in range(nst - 1)) if nst > 1 else np.zeros((d, d))
                M_d = sum(blk(t + 1, t) + np.outer(mu[t + 1] - uu, mu[t]) for t in range(nst - 1)) if nst > 1 else np.zeros((d, d))
                Lmat = np.concatenate([-An[c], np.eye(d)], axis=1)
                R_d = K_new[c].copy()
                for t in range(nst - 1):
                    e = mu[t + 1] - An[c] @ mu[t] - uu
                    R_d += Lmat @ Sig[t * d:(t + 2) * d, t * d:(t + 2) * d] @ Lmat.T + np.outer(e, e)
                dense["Lam"].append(Va0i + np.kron(Wp[c], Sxx_d)); dense["xi"].append(Va0i @ ma0 + (Wp[c] @ M_d).reshape(n))
                dense["R_new"].append(R_d)
            hist["stats"].append(dict(Lam=Lam, xi=xi, R_new=R_new, R_update_form=R_upd,
                                      **{k + "_dense": np.stack(v) for k, v in dense.items()}))
        # ---- q(w_p) with the new q(a), q(w_q)
        qp = qq = None
        if lp:
            nu0, Psi0 = float(p_prior[0]), np.asarray(p_prior[1], np.float64)
            df = np.full(batch, nu0 + Np); Psi = Psi0[None] + R_new
            fe = fe + sum(_wishart_block(Np, Wp, df, Psi, nu0, Psi0, R_new))
            Wpn = df[:, None, None] * np.linalg.inv(Psi)
            Wpn = 0.5 * (Wpn + np.swapaxes(Wpn, -1, -2))
            qp = (df, Psi, nu0, Psi0)
            hist["df_p"].append(df); hist["inv_scale_p"].append(np.moveaxis(Psi, 0, 2)); hist["E_Wp"].append(np.moveaxis(Wpn, 0, 2))
        if lq:
            o = 1 if tf else 0
            mu_o, S_o = sm[o:], sS[o:]
            e = yb - np.einsum("ij,tbj->tbi", B, mu_o)
            terms = np.einsum("tbi,tbj->tbij", e, e) + np.einsum("ij,tbjk,lk->tbil", B, S_o, B)
            Rq = np.where(mk[..., None, None], terms, 0.0).sum(0)
            nobs = mk.sum(0)
            nu0, Psi0 = float(q_prior[0]), np.asarray(q_prior[1], np.float64)
            df = nu0 + nobs.astype(np.float64); Psi = Psi0[None] + Rq
            Wqn = df[:, None, None] * np.linalg.inv(Psi)
            Wqn = 0.5 * (Wqn + np.swapaxes(Wqn, -1, -2))
            Elog = _mvdigamma(0.5 * df, m) + m * np.log(2.0) - np.linalg.slogdet(Psi)[1]
            fe = (fe + 0.5 * nobs * (np.linalg.slogdet(Wq)[1] - Elog) + 0.5 * np.einsum("bij,bji->b", Wqn - Wq, Rq)
                  + wishart_kl(df, Psi, nu0, Psi0))
            qq = (df, Psi, nu0, Psi0)
            hist["df_q"].append(df); hist["inv_scale_q"].append(np.moveaxis(Psi, 0, 2)); hist["E_Wq"].append(np.moveaxis(Wqn, 0, 2))
        if definition:
            hist["free_energy_definition"].append(_definition(
                yb, mk, Abar, Wp, Wq, Xi, B, m0, S0, uu, tf, P, Q, qp, qq, am_n, Sa_n, ma0, Va0))
        hist["free_energy"].append(fe)
        hist["a_mean"].append(np.moveaxis(An, 0, 2)); hist["a_cov"].append(np.moveaxis(Sa_n, 0, 2))
        am, Sa = am_n, Sa_n
        if lp:
            Wp = Wpn
        if lq:
            Wq = Wqn
    out = {k: np.stack(v) for k, v in hist.items() if v and k != "stats"}
    out["stats"] = hist["stats"]
    o = 1 if tf else 0
    out["mean"] = np.transpose(r["mean"][o:], (0, 2, 1))
    out["cov"] = np.transpose(r["cov"][o:], (0, 2, 3, 1))
    return out


def _definition(yb, mk, Abar, Wp_old, Wq_old, Xi, B, m0, S0, u, tf, P, Q, qp, qq, am, Sa, ma0, Va0):
    """F = E_q[-log p(y, x, a, w_p, w_q)] - H[q(x)] - H[q(a)] - H[q(w_p)] - H[q(w_q)], one chain at a time: q(x) the dense
    posterior the sweep computed (under the previous q(a), q(w)), the expectations over the new q(a), q(w) in closed form:
    E_q(a)[(x' - A x - u)(...)'] = (x' - Abar x - u)(...)' + E[(A - Abar) x x' (A - Abar)']."""
    T, batch, m = yb.shape
    d = Abar.shape[-1]
    n = d * d
    out = np.zeros(batch)
    for c in range(batch):
        mu, Sig = _dense_chain(yb[:, c], mk[:, c], Abar[c], Wp_old[c], Wq_old[c], Xi[c], B, m0, S0, u, tf)
        nst = mu.shape[0]
        o = 1 if tf else 0
        S0i = np.linalg.inv(S0)
        dm = mu[0] - m0
        F = 0.5 * (d * np.log(2 * np.pi) + np.linalg.slogdet(S0)[1] + np.trace(S0i @ Sig[:d, :d]) + dm @ S0i @ dm)
        A = am[c].reshape(d, d)
        Lmat = np.concatenate([-A, np.eye(d)], axis=1)
        Rp = np.zeros((d, d)); Sxx = np.zeros((d, d))
        for t in range(nst - 1):
            e = mu[t + 1] - A @ mu[t] - u
            Rp += Lmat @ Sig[t * d:(t + 2) * d, t * d:(t + 2) * d] @ Lmat.T + np.outer(e, e)
            Sxx += Sig[t * d:(t + 1) * d, t * d:(t + 1) * d] + np.outer(mu[t], mu[t])
        Rp += _kron_contract(Sa[c][None], Sxx[None], d)[0]
        Np = nst - 1
        if qp is None:
            F += 0.5 * (Np * d * np.log(2 * np.pi) + Np * np.linalg.slogdet(P)[1] + np.trace(np.linalg.inv(P) @ Rp))
        else:
            df, Psi, nu0, Psi0 = qp
            Ew, Elog, E_pw, H_w = _Ew_terms(df[c], Psi[c], nu0, Psi0)
            F += 0.5 * (Np * d * np.log(2 * np.pi) - Np * Elog + np.trace(Ew @ Rp)) + E_pw - H_w
        Rq = np.zeros((m, m)); nq = 0
        for t in range(T):
            if mk[t, c]:
                s = slice((t + o) * d, (t + o + 1) * d)
                e = yb[t, c] - B @ mu[t + o]
                Rq += np.outer(e, e) + B @ Sig[s, s] @ B.T
                nq += 1
        if qq is None:
            F += 0.5 * (nq * m * np.log(2 * np.pi) + nq * np.linalg.slogdet(Q)[1] + np.trace(np.linalg.inv(Q) @ Rq))
        else:
            df, Psi, nu0, Psi0 = qq
            Ew, Elog, E_pw, H_w = _Ew_terms(df[c], Psi[c], nu0, Psi0)
            F += 0.5 * (nq * m * np.log(2 * np.pi) - nq * Elog + np.trace(Ew @ Rq)) + E_pw - H_w
        F -= 0.5 * (nst * d * (1 + np.log(2 * np.pi)) + np.linalg.slogdet(Sig)[1])
        # E_q(a)[-log p(a)] - H[q(a)]
        Vi = np.linalg.inv(Va0)
        da = am[c] - ma0
        F += 0.5 * (n * np.log(2 * np.pi) + np.linalg.slogdet(Va0)[1] + np.trace(Vi @ Sa[c]) + da @ Vi @ da)
        F -= 0.5 * (n * (1 + np.log(2 * np.pi)) + np.linalg.slogdet(Sa[c])[1])
        out[c] = F
    return out


# ====================================================================================== problems
def a_prior(d, A=None, scale=1.0):
    """N(vec(A) or 0, scale I) (row-major)."""
    return (np.zeros(d * d) if A is None else np.asarray(A, np.float64).reshape(-1)), scale * np.eye(d * d)


def a_init(A, scale=0.01):
    """q(a) started at E[A] = A with a small covariance that couples the entries of each row."""
    d = A.shape[0]
    n = d * d
    C = np.eye(n) * scale
    for i in range(d):
        for j in range(d - 1):
            C[i * d + j, i * d + j + 1] = C[i * d + j + 1, i * d + j] = 0.3 * scale
    return np.asarray(A, np.float64).reshape(-1), C


def mode_kwargs(mod, mode, d, m):
    """Noise arguments for mode "A", "AP", "AQ" or "APQ"."""
    kw = {}
    if "P" in mode:
        kw.update(p_prior=(float(d + 2), np.eye(d) * 0.2), p_init=np.linalg.inv(mod["P"]))
    else:
        kw["P"] = mod["P"]
    if "Q" in mode:
        kw.update(q_prior=(float(m + 2), np.eye(m) * 0.5), q_init=np.eye(m) * 1.5)
    else:
        kw["Q"] = np.eye(m) * 0.5
    return kw


def problem(d, m, T, batch, seed):
    """random_problem plus the A prior (centred at a perturbation of the true A) and an initial q(a) at the true A."""
    mod, y, _, _ = random_problem(d, m, T, batch, seed=seed)
    rng = np.random.default_rng(seed + 1)
    ma0 = mod["A"] + 0.1 * rng.standard_normal((d, d))
    pri = (ma0.reshape(-1), 0.5 * np.eye(d * d))
    return mod, y, pri, a_init(mod["A"] + 0.05 * rng.standard_normal((d, d)), 0.02)


def _mask(kind, T, batch):
    if kind is None:
        return None
    if kind == "shared":
        mk = np.ones(T, dtype=np.uint8); mk[0] = 0; mk[-1] = 0
        return mk
    mk = np.ones((T, batch), dtype=np.uint8)
    mk[0, 0] = 0; mk[-1, 1] = 0; mk[2:4, 2] = 0
    mk[:, -1] = 0                                         # a chain with no observation
    return mk


# ====================================================================================== closed form vs definition
FE_CASES = [(mode, d, m, tf, with_u, mk) for mode in MODES for (d, m, tf, with_u, mk) in
            [(1, 1, False, False, None), (2, 3, True, True, "gaps"), (3, 2, True, False, "shared"), (2, 1, False, True, "gaps")]]


@pytest.mark.parametrize("mode,d,m,tf,with_u,mask", FE_CASES)
def test_closed_form_free_energy_equals_the_definition(mode, d, m, tf, with_u, mask):
    """Every mode, (d, m) with m > d and m < d, masks with the first and last step missing and an all-missing chain,
    transition_first and a constant u: the closed-form F equals the definition (dense joint q(x), closed-form expectations
    over q(a) and q(w)) to 1e-10; Lambda_a, xi_a and R_p at the new E[A] from the pair statistics equal the dense-joint
    values, and so does the kernel's update form of R_p, to 1e-10."""
    T, batch = 6, 4
    mod, y, pri, ini = problem(d, m, T, batch, seed=30 * d + m + (7 if tf else 0))
    u = np.linspace(-0.3, 0.4, d) if with_u else None
    r = lgssm_continuous_transition(y, mod["B"], mod["m0"], mod["S0"], 4, a_prior=pri, a_init=ini,
                                    mask=_mask(mask, T, batch), u=u, transition_first=tf, definition=True, stats_check=True,
                                    **mode_kwargs(mod, mode, d, m))
    fe, fd = r["free_energy"], r["free_energy_definition"]
    assert np.abs(fe - fd).max() <= 1e-10 * max(1.0, np.abs(fd).max()), np.abs(fe - fd).max()
    for st in r["stats"]:
        for k in ("Lam", "xi", "R_new"):
            scale = np.abs(st[k + "_dense"]).max()
            assert np.abs(st[k] - st[k + "_dense"]).max() <= 1e-10 * scale, k
        assert np.abs(st["R_update_form"] - st["R_new"]).max() <= 1e-10 * np.abs(st["R_new"]).max()


@pytest.mark.parametrize("mode", ["AP", "AQ", "APQ"])
def test_a_known_to_the_precision_is_the_noise_reference(mode):
    """a_cov0 = a_init_cov = 1e-10 I around a fixed A: q(a) cannot move, Xi vanishes and the result tends to the
    reference with A known (test_vmp_noise.lgssm_wishart_noise)."""
    d, m, T, batch = 2, 3, 12, 4
    mod, y, _, _ = random_problem(d, m, T, batch, seed=11)
    pri = (mod["A"].reshape(-1), 1e-10 * np.eye(d * d))
    kw = mode_kwargs(mod, mode, d, m)
    r = lgssm_continuous_transition(y, mod["B"], mod["m0"], mod["S0"], 5, a_prior=pri, a_init=pri,
                                    mask=_mask("gaps", T, batch), transition_first=True, **kw)
    ref = lgssm_wishart_noise(y, mod["A"], mod["B"], mod["m0"], mod["S0"], 5, mask=_mask("gaps", T, batch),
                              transition_first=True, **kw)
    for k in ("mean", "cov", "inv_scale_p", "inv_scale_q", "free_energy"):
        if k in ref:
            assert np.abs(r[k] - ref[k]).max() <= 1e-6 * max(1.0, np.abs(ref[k]).max()), k
    assert np.abs(r["a_mean"] - mod["A"][None, :, :, None]).max() <= 1e-8


@pytest.mark.parametrize("mode", MODES)
def test_single_step_without_transition_keeps_the_prior(mode):
    d, m, batch = 2, 2, 3
    mod, y, pri, ini = problem(d, m, 1, batch, seed=4)
    r = lgssm_continuous_transition(y, mod["B"], mod["m0"], mod["S0"], 3, a_prior=pri, a_init=ini, definition=True,
                                    **mode_kwargs(mod, mode, d, m))
    assert np.allclose(r["a_mean"], pri[0].reshape(d, d)[None, :, :, None], rtol=0, atol=1e-14)
    assert np.allclose(r["a_cov"], pri[1][None, :, :, None], rtol=0, atol=1e-14)
    assert np.abs(r["free_energy"] - r["free_energy_definition"]).max() <= 1e-10 * max(1.0, np.abs(r["free_energy"]).max())


@pytest.mark.parametrize("mode", MODES)
def test_free_energy_is_non_increasing_over_30_iterations(mode):
    T, batch, d, m = 40, 5, 3, 2
    mod, y, pri, ini = problem(d, m, T, batch, seed=7)
    r = lgssm_continuous_transition(y, mod["B"], mod["m0"], mod["S0"], 30, a_prior=pri, a_init=ini,
                                    mask=_mask("gaps", T, batch), transition_first=True, u=np.linspace(-0.2, 0.1, d),
                                    **mode_kwargs(mod, mode, d, m))
    fe = r["free_energy"]
    assert np.all(np.diff(fe, axis=0) <= 1e-9 * np.abs(fe[1:]))


def test_posterior_mean_recovers_the_true_transition_matrix():
    """T = 2000 draws from a stable non-symmetric A with B = I and a small Q: E[A] is within 5 posterior standard
    deviations of the truth, entry by entry (A, P and Q learned)."""
    T, batch, d = 2000, 3, 2
    rng = np.random.default_rng(41)
    A = np.array([[0.8, 0.3], [-0.4, 0.7]])
    P = np.array([[0.3, 0.05], [0.05, 0.2]])
    LP = np.linalg.cholesky(P)
    y = np.zeros((T, d, batch))
    for c in range(batch):
        x = rng.standard_normal(d)
        for t in range(T):
            if t > 0:
                x = A @ x + LP @ rng.standard_normal(d)
            y[t, :, c] = x + np.sqrt(1e-3) * rng.standard_normal(d)
    r = lgssm_continuous_transition(y, np.eye(d), np.zeros(d), np.eye(d), 10, a_prior=a_prior(d), a_init=a_init(np.eye(d) * 0.5, 0.1),
                                    p_prior=(d + 2.0, 0.1 * np.eye(d)), p_init=np.eye(d), q_prior=(d + 2.0, 1e-3 * np.eye(d)),
                                    q_init=1e3 * np.eye(d))
    for c in range(batch):
        sd = np.sqrt(np.diag(r["a_cov"][-1][:, :, c])).reshape(d, d)
        assert np.all(np.abs(r["a_mean"][-1][:, :, c] - A) <= 5 * sd), (r["a_mean"][-1][:, :, c], sd)


def conditioning_problem(batch=4, T=400, seed=3):
    """Large states (|x| ~ 1e3: a slowly drifting A close to a rotation, a large prior mean) and a small process noise
    (P = 1e-4 I) observed precisely: the second moments of x are ~1e6 times R_p / N_p."""
    d = m = 2
    rng = np.random.default_rng(seed)
    th = 0.05
    A = 0.999 * np.array([[np.cos(th), -np.sin(th)], [np.sin(th), np.cos(th)]])
    P = 1e-4 * np.eye(d)
    y = np.zeros((T, m, batch))
    for c in range(batch):
        x = np.array([1500.0, -800.0]) + rng.standard_normal(d)
        for t in range(T):
            if t > 0:
                x = A @ x + 1e-2 * rng.standard_normal(d)
            y[t, :, c] = x + 1e-2 * rng.standard_normal(m)
    f32 = lambda M: np.asarray(M, np.float32).astype(np.float64)
    mod = dict(A=f32(A), B=np.eye(d), P=f32(P), m0=f32([1500.0, -800.0]), S0=np.eye(d) * 4.0, Q=np.eye(m) * 1e-4)
    return mod, y.astype(np.float32)


def test_conditioning_of_the_residual_form():
    """Large states and a small P: R_p at the new E[A] in the kernel's update form, with every per-step term rounded to
    fp32 before the fp64 sum (as the kernel folds them), stays within 1e-5 of the fp64 pair-covariance value, while the
    second-moment form S_yy - A S_xy' - S_xy A' + A S_xx A' with the same fp32 terms loses all accuracy."""
    mod, y = conditioning_problem()
    d = 2
    kw = dict(p_prior=(d + 2.0, 1e-4 * np.eye(d)), p_init=np.linalg.inv(mod["P"]), Q=mod["Q"])
    pri = (mod["A"].reshape(-1), 1e-2 * np.eye(d * d))
    ini = (mod["A"].reshape(-1) + 1e-3, 1e-6 * np.eye(d * d))
    r = lgssm_continuous_transition(y, mod["B"], mod["m0"], mod["S0"], 2, a_prior=pri, a_init=ini, stats_check=True, **kw)
    # rebuild the statistics of the last sweep with fp32 per-step terms
    yb = np.transpose(np.asarray(y, np.float64), (0, 2, 1))
    st = r["stats"][-1]
    Abar = r["a_mean"][0].transpose(2, 0, 1)                  # E[A] the last sweep used
    An = r["a_mean"][1].transpose(2, 0, 1)
    Sa_last = r["a_cov"][0].transpose(2, 0, 1)
    Wp = r["E_Wp"][0].transpose(2, 0, 1)
    Lx = np.linalg.cholesky(_xi(Sa_last, Wp, d))
    sm_ = tilted_smoother(yb, np.ones(yb.shape[:2], bool), Abar, np.linalg.inv(Wp), np.broadcast_to(mod["Q"], (4, d, d)),
                          mod["B"], mod["m0"], mod["S0"], np.zeros(d), False, Lx)
    sm, sS, cross = sm_["mean"], sm_["cov"], sm_["cross"]
    r32 = lambda a: np.asarray(a, np.float32).astype(np.float64)
    At = np.swapaxes(Abar, -1, -2)
    R_old = Sxx = Sxr = Syy = Sxy = 0.0
    for t in range(sm.shape[0] - 1):
        C = cross[t]
        V = sS[t + 1] - C @ At - Abar @ np.swapaxes(C, -1, -2) + Abar @ sS[t] @ At
        e = sm[t + 1] - np.einsum("bij,bj->bi", Abar, sm[t])
        R_old = R_old + r32(V + np.einsum("bi,bj->bij", e, e))
        Sxx = Sxx + r32(sS[t] + np.einsum("bi,bj->bij", sm[t], sm[t]))
        Sxr = Sxr + r32(np.swapaxes(C, -1, -2) - sS[t] @ At + np.einsum("bi,bj->bij", sm[t], e))
        Syy = Syy + r32(sS[t + 1] + np.einsum("bi,bj->bij", sm[t + 1], sm[t + 1]))
        Sxy = Sxy + r32(C + np.einsum("bi,bj->bij", sm[t + 1], sm[t]))
    Dl = An - Abar
    K_new = st["R_new"] - residual_R(sm, sS, cross, An, np.zeros(d))
    R_upd = R_old + Dl @ Sxx @ np.swapaxes(Dl, -1, -2) - Dl @ Sxr - np.swapaxes(Sxr, -1, -2) @ np.swapaxes(Dl, -1, -2) + K_new
    Ant = np.swapaxes(An, -1, -2)
    R_mom = Syy - Sxy @ Ant - An @ np.swapaxes(Sxy, -1, -2) + An @ Sxx @ Ant + K_new
    rel = lambda a: np.linalg.norm(a - st["R_new"], axis=(1, 2)) / np.linalg.norm(st["R_new"], axis=(1, 2))
    assert rel(R_upd).max() <= 1e-5, rel(R_upd)
    assert rel(R_mom).min() >= 1e-2, rel(R_mom)


# ====================================================================================== argument handling (no device)
def _bare_context():
    from rxinfer_jl_b200.context import Context
    return object.__new__(Context)


def test_context_argument_rules(rx):
    c = _bare_context()
    mod, y, pri, ini = problem(2, 2, 5, 3, seed=1)
    y = torch.as_tensor(y)
    args = (mod["B"], mod["m0"], mod["S0"])
    kw = dict(a_prior=pri, a_init=ini, P=mod["P"], Q=np.eye(2))
    with pytest.raises(TypeError, match="a_init"):
        c.lgssm_vmp_transition(y, *args, a_prior=pri, P=mod["P"], Q=np.eye(2))          # no initial q(a)
    with pytest.raises(ValueError, match="a_init: expected"):
        c.lgssm_vmp_transition(y, *args, **dict(kw, a_init=pri[0]))
    with pytest.raises(ValueError, match="a_cov0: expected shape"):
        c.lgssm_vmp_transition(y, *args, **dict(kw, a_prior=(pri[0], np.eye(3))))
    with pytest.raises(ValueError, match="a_init_mean: expected shape"):
        c.lgssm_vmp_transition(y, *args, **dict(kw, a_init=(np.zeros(3), ini[1])))
    with pytest.raises(ValueError, match="P is learned: pass p_prior"):
        c.lgssm_vmp_transition(y, *args, a_prior=pri, a_init=ini, Q=np.eye(2), p_prior=(4.0, np.eye(2)))
    with pytest.raises(ValueError, match="iterations must be >= 1"):
        c.lgssm_vmp_transition(y, *args, **kw, iterations=0)
    with pytest.raises(ValueError, match="expected \\[T, m, batch\\]"):
        c.lgssm_vmp_transition(y[0], *args, **kw)
    c.device = 0
    with pytest.raises(ValueError, match="y: expected a tensor on cuda"):
        c.lgssm_vmp_transition(y, *args, **kw)                       # both noises known is accepted up to here


def test_vec_order_round_trip(rx):
    """vec_order maps Julia's column-major vec(A) to the ABI's row-major a and back."""
    from rxinfer_jl_b200.inference import vec_order
    for d in (1, 2, 3, 4):
        A = np.arange(d * d, dtype=np.float64).reshape(d, d) * 1.5 - 2.0
        col = A.reshape(-1, order="F")                                 # Julia vec(A)
        p = vec_order(d)
        assert np.array_equal(col[p], A.reshape(-1)) and np.array_equal(A.reshape(-1)[p], col)
        V = np.outer(col, col) + np.diag(np.arange(d * d) + 1.0)     # cov over vec(A)
        Vr = V[np.ix_(p, p)]
        for i in range(d * d):
            for j in range(d * d):
                assert Vr[i, j] == V[p[i], p[j]]
        assert np.array_equal(Vr[np.ix_(p, p)], V)


def test_infer_argument_rules(rx):
    from rxinfer_jl_b200 import inference as I
    mod, _, pri, ini = problem(2, 2, 5, 3, seed=1)
    model = I.linear_gaussian_ssm_continuous_transition(B=mod["B"], x0=(mod["m0"], mod["S0"]), a_prior=pri, a_init=ini,
                                                        P=mod["P"], Q=np.eye(2))
    y = torch.zeros(5, 2, 3)
    with pytest.raises(NotImplementedError, match="input sequences"):
        I.infer(model=model, data={"y": y, "u": np.zeros((5, 2))}, iterations=3)
    with pytest.raises(NotImplementedError, match="predictions"):
        I.infer(model=model, data={"y": y}, iterations=3, predictvars={"y": I.KeepLast()})
    with pytest.raises(NotImplementedError, match="KeepLast"):
        I.infer(model=model, data={"y": y}, iterations=3, returnvars={"x": I.KeepEach()})
    with pytest.raises(ValueError, match="needs `data`"):
        I.infer(model=model, iterations=3)
    no_init = I.linear_gaussian_ssm_continuous_transition(B=mod["B"], x0=(mod["m0"], mod["S0"]), a_prior=pri,
                                                          P=mod["P"], Q=np.eye(2))
    with pytest.raises(ValueError, match="a_init"):
        I.infer(model=no_init, data={"y": y}, iterations=3, context=_bare_context())


def _shim():
    import os
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    return open(os.path.join(root, "rxinfer.jl_b200", "julia", "RxGaussB200.jl")).read()


def test_julia_helper_packs_the_call():
    """`lgssm_continuous_transition(ctx, y; ...)` requires a_init, permutes vec(A) (column-major) to the ABI's row-major
    order on the way in and back on the way out, passes NULL for what a known noise does not have and an fp64
    free-energy buffer."""
    s = _shim()
    body = s[s.index("function lgssm_continuous_transition(ctx::Context"):]
    body = body[:body.index("\nend\n")]
    assert "batch, m, T = size(y)" in body and "a_init === nothing && throw" in body
    assert "p = vec(permutedims(reshape(1:n, d, d)))" in body
    assert "vec(a_prior[1])[p]" in body and "a_prior[2][p, p]" in body and "a_init[2][p, p]" in body
    assert "download(am)[:, p, :], download(aV)[:, p, p, :]" in body
    assert "Lib.lgssm_vmp_transition(ctx, d, m, T, batch," in body
    assert "ptr(Pt), nup, ptr(iSp0), ptr(EWp0), ptr(Qt), nuq, ptr(iSq0), ptr(EWq0)" in body
    assert "reinterpret(Float64" in body and "RXG_TRANSITION_FIRST" in body
    # the Julia index map is the Python one (1-based)
    from importlib import import_module
    for d in (2, 3, 4):
        jl = np.arange(1, d * d + 1).reshape(d, d, order="F").T.reshape(-1, order="F")    # vec(permutedims(reshape(1:n, d, d)))
        assert np.array_equal(jl - 1, import_module("rxinfer_jl_b200.inference").vec_order(d))
