"""fp64 reference of the VMP with an unknown process precision matrix (rxg_lgssm_vmp_noise_f32), alone or together with the
observation precision, and its CPU checks.

Model (per chain): w_p ~ Wishart(nu_p0, inv(Psi_p0)) (else P known); w_q ~ Wishart(nu_q0, inv(Psi_q0)) (else Q known);
x[1] ~ N(m0, S0) (or one transition earlier); x[t] ~ N(A x[t-1] + u, inv(w_p)); y[t] ~ N(B x[t], inv(w_q));
q(x) q(w_p) q(w_q).  ``lgssm_wishart_noise`` runs the schedule message by message:
  q(x)   oracle.lgssm.smooth_reference_schedule with the per-chain P = inv(E[w_p]) and Q = inv(E[w_q]);
  q(w_q) folded exactly as test_vmp_wishart.lgssm_wishart_precision folds it;
  q(w_p) the prior folded with one MvNormalMeanPrecision(:Lambda) message per transition, Wishart(d + 2, inv(R_t)) with
         R_t = E[(x_{t+1} - A x_t - u)(x_{t+1} - A x_t - u)'] under the pairwise marginal of the transition node, built from
         the messages around it (filtered state at t, transition factor, observation and backward message at t + 1);
  F      the Bethe free energy in closed form (what the kernel evaluates) and, with ``definition=True``, from its definition
         with a dense Gaussian q(x) over every latent state (x_0 included with transition_first).
"""
import numpy as np
import pytest
import torch

from oracle import lgssm, rules as R
from test_vmp_wishart import _mvdigamma, _mvlgamma, random_problem, wishart_kl


def _pair_stat(L, mu, Sig, u):
    """E[(L z - u)(L z - u)'] for z ~ N(mu, Sig), batched."""
    e = np.einsum("ij,bj->bi", L, mu) - u
    return np.einsum("ij,bjk,lk->bil", L, Sig, L) + np.einsum("bi,bj->bij", e, e)


def _pair_messages(r, A, Pb, m0, S0, u, tf):
    """R_p from the pairwise marginal of every transition node, message by message: the filtered state at t (the prior
    (m0, S0) for the transition into x[1] with transition_first), the transition N(x' | A x + u, P) and the product of the
    observation and backward messages at t + 1.  Returns the per-transition terms [N_p, batch, d, d]."""
    T, batch, d = r["fwd_mean"].shape
    fm = np.transpose(r["filt_mean"], (0, 2, 1)); fS = np.transpose(r["filt_cov"], (0, 3, 1, 2))
    Lam = np.linalg.inv(Pb)
    Lmat = np.concatenate([-A, np.eye(d)], axis=1)
    starts = ([(np.broadcast_to(m0, (batch, d)), np.broadcast_to(S0, (batch, d, d)), 0)] if tf else []) + \
             [(fm[t], fS[t], t + 1) for t in range(T - 1)]
    out = []
    for mf, Sf, t1 in starts:
        Jf = np.linalg.inv(Sf); hf = np.einsum("bij,bj->bi", Jf, mf)
        xi_b = r["obs_xi"][t1] + r["bwd_xi"][t1]; W_b = r["obs_W"][t1] + r["bwd_W"][t1]
        LA = Lam @ A
        J = np.zeros((batch, 2 * d, 2 * d)); h = np.zeros((batch, 2 * d))
        J[:, :d, :d] = Jf + np.swapaxes(A, -1, -2) @ LA
        J[:, :d, d:] = -np.swapaxes(LA, -1, -2)
        J[:, d:, :d] = -LA
        J[:, d:, d:] = Lam + W_b
        Lu = np.einsum("bij,j->bi", Lam, u)
        h[:, :d] = hf - np.einsum("ji,bj->bi", A, Lu)
        h[:, d:] = Lu + xi_b
        Sig = np.linalg.inv(J); mu = np.einsum("bij,bj->bi", Sig, h)
        out.append(_pair_stat(Lmat, mu, Sig, u))
    return np.stack(out) if out else np.zeros((0, batch, d, d))


def pair_form_Rp(r, A, Pb, m0, S0, u, tf):
    """R_p as the kernel forms it, in fp64: with the RTS gain G_t = Sf A' Sp^-1 and C_t = Sf - G_t Sp G_t',
    cov(x_{t+1} - A x_t | y) = (I - A G_t) Sigma_s[t+1] (I - A G_t)' + A C_t A', plus e e', e = mu_s[t+1] - A mu_s[t] - u;
    with transition_first one more RTS step from (m0, S0) into x[1]."""
    T, batch, d = r["fwd_mean"].shape
    fm = np.transpose(r["filt_mean"], (0, 2, 1)); fS = np.transpose(r["filt_cov"], (0, 3, 1, 2))
    sm = np.transpose(r["mean"], (0, 2, 1)); sS = np.transpose(r["cov"], (0, 3, 1, 2))
    I = np.eye(d)
    starts = ([(np.broadcast_to(m0, (batch, d)), np.broadcast_to(S0, (batch, d, d)), 0)] if tf else []) + \
             [(fm[t], fS[t], t + 1) for t in range(T - 1)]
    Rp = np.zeros((batch, d, d))
    for mf, Sf, t1 in starts:
        Sp = A @ Sf @ A.T + Pb
        G = Sf @ A.T @ np.linalg.inv(Sp)
        C = Sf - G @ Sp @ np.swapaxes(G, -1, -2)
        F = I - A @ G
        ms = mf + np.einsum("bij,bj->bi", G, sm[t1] - np.einsum("ij,bj->bi", A, mf) - u)   # smoothed at t
        e = sm[t1] - np.einsum("ij,bj->bi", A, ms) - u
        Rp += F @ sS[t1] @ np.swapaxes(F, -1, -2) + A @ C @ A.T + np.einsum("bi,bj->bij", e, e)
    return Rp


def _wishart_block(n, W, df, Psi, nu0, Psi0, Rsum):
    """n/2 (log det Wbar - E log det w) + 1/2 tr((E w - Wbar) R) + KL(q(w) || prior), as three terms (left to right)."""
    k = Psi.shape[-1]
    Wn = df[:, None, None] * np.linalg.inv(Psi)
    Elog = _mvdigamma(0.5 * df, k) + k * np.log(2.0) - np.linalg.slogdet(Psi)[1]
    return (0.5 * n * (np.linalg.slogdet(W)[1] - Elog), 0.5 * np.einsum("bij,bji->b", Wn - W, Rsum),
            wishart_kl(df, Psi, float(nu0), Psi0))


def _Ew_terms(df, Psi, nu0, Psi0):
    """E[w], E log det w, E_q[-log p(w)] and H[q(w)] of one chain's Wishart(df, inv(Psi))."""
    k = Psi.shape[-1]
    Ew = df * np.linalg.inv(Psi)
    ld_S = -np.linalg.slogdet(Psi)[1]
    Elog = _mvdigamma(0.5 * df, k) + k * np.log(2.0) + ld_S
    E_pw = (-0.5 * (nu0 - k - 1) * Elog + 0.5 * np.trace(Psi0 @ Ew) + 0.5 * nu0 * k * np.log(2.0)
            - 0.5 * nu0 * np.linalg.slogdet(Psi0)[1] + _mvlgamma(0.5 * nu0, k))
    H_w = 0.5 * df * ld_S + 0.5 * df * k * np.log(2.0) + _mvlgamma(0.5 * df, k) - 0.5 * (df - k - 1) * Elog + 0.5 * df * k
    return Ew, Elog, E_pw, H_w


def dense_posterior(y, mk, A, B, m0, S0, u, tf, Lam, Wq, c):
    """Dense Gaussian q(x) of chain c over (x_0,) x_1..x_T under transition precision Lam[c] and observation precision
    Wq[c]; returns (mu, Sig, n_states, offset of x_1)."""
    T, m, _ = y.shape
    d = A.shape[0]
    n = T + (1 if tf else 0)
    o = 1 if tf else 0
    J = np.zeros((n * d, n * d)); h = np.zeros(n * d)
    S0i = np.linalg.inv(S0)
    J[:d, :d] += S0i; h[:d] += S0i @ m0
    Li = Lam[c]
    for t in range(1, n):
        a, b = slice((t - 1) * d, t * d), slice(t * d, (t + 1) * d)
        J[b, b] += Li; J[a, a] += A.T @ Li @ A
        J[b, a] -= Li @ A; J[a, b] -= A.T @ Li
        h[b] += Li @ u; h[a] -= A.T @ Li @ u
    for t in range(T):
        if mk[t, c]:
            s = slice((t + o) * d, (t + o + 1) * d)
            J[s, s] += B.T @ Wq[c] @ B
            h[s] += B.T @ Wq[c] @ y[t, :, c]
    Sig = np.linalg.inv(J)
    return Sig @ h, Sig, n, o


def dense_Rp(mu, Sig, n, A, u):
    d = A.shape[0]
    Lmat = np.concatenate([-A, np.eye(d)], axis=1)
    Rp = np.zeros((d, d))
    for t in range(1, n):
        s = slice((t - 1) * d, (t + 1) * d)
        Rp += _pair_stat(Lmat, mu[None, s], Sig[None, s, s], u)[0]
    return Rp


def _free_energy_definition(y, mk, A, B, m0, S0, u, tf, Pk, Qk, Wp, Wq, qp, qq):
    """F = E_q[-log p(y, x, w_p, w_q)] - H[q(x)] - H[q(w_p)] - H[q(w_q)] with q(x) the exact posterior under
    (Wbar_p, Wbar_q), one chain at a time with dense algebra over every latent state.  qp / qq: (df, Psi, nu0, Psi0) of a
    learned noise or None (then Pk / Qk is the known covariance)."""
    T, m, batch = y.shape
    d = A.shape[0]
    out = np.zeros(batch)
    Lam = np.broadcast_to(np.linalg.inv(Pk), (batch, d, d)) if qp is None else Wp
    Wobs = np.broadcast_to(np.linalg.inv(Qk), (batch, m, m)) if qq is None else Wq
    for c in range(batch):
        mu, Sig, n, o = dense_posterior(y, mk, A, B, m0, S0, u, tf, Lam, Wobs, c)
        S0i = np.linalg.inv(S0)
        dm = mu[:d] - m0
        F = 0.5 * (d * np.log(2 * np.pi) + np.linalg.slogdet(S0)[1] + np.trace(S0i @ Sig[:d, :d]) + dm @ S0i @ dm)
        Rp = dense_Rp(mu, Sig, n, A, u)
        Np = n - 1
        if qp is None:
            F += 0.5 * (Np * d * np.log(2 * np.pi) + Np * np.linalg.slogdet(Pk)[1] + np.trace(np.linalg.inv(Pk) @ Rp))
        else:
            df, Psi, nu0, Psi0 = qp
            Ew, Elog, E_pw, H_w = _Ew_terms(df[c], Psi[c], nu0, Psi0)
            F += 0.5 * (Np * d * np.log(2 * np.pi) - Np * Elog + np.trace(Ew @ Rp)) + E_pw - H_w
        Rq = np.zeros((m, m)); nq = 0
        for t in range(T):
            if mk[t, c]:
                s = slice((t + o) * d, (t + o + 1) * d)
                e = y[t, :, c] - B @ mu[s]
                Rq += np.outer(e, e) + B @ Sig[s, s] @ B.T
                nq += 1
        if qq is None:
            F += 0.5 * (nq * m * np.log(2 * np.pi) + nq * np.linalg.slogdet(Qk)[1] + np.trace(np.linalg.inv(Qk) @ Rq))
        else:
            df, Psi, nu0, Psi0 = qq
            Ew, Elog, E_pw, H_w = _Ew_terms(df[c], Psi[c], nu0, Psi0)
            F += 0.5 * (nq * m * np.log(2 * np.pi) - nq * Elog + np.trace(Ew @ Rq)) + E_pw - H_w
        F -= 0.5 * (n * d * (1 + np.log(2 * np.pi)) + np.linalg.slogdet(Sig)[1])
        out[c] = F
    return out


def lgssm_wishart_noise(y, A, B, m0, S0, iterations, *, P=None, Q=None, p_prior=None, p_init=None, q_prior=None,
                        q_init=None, mask=None, u=None, transition_first=False, definition=False, pair_check=False):
    """y[T, m, batch]; mask None, [T, batch] or a shared [T] pattern.  Returns dict(mean[T, d, batch], cov[T, d, d, batch]
    of the last iteration; df_p / inv_scale_p / E_Wp and df_q / inv_scale_q / E_Wq per iteration for the learned noises
    ([iterations, batch] / [iterations, k, k, batch]); free_energy[iterations, batch] (closed form) and, with
    ``definition``, free_energy_definition; with ``pair_check``, Rp_messages / Rp_pair_form / Rp_dense per iteration)."""
    y = np.asarray(y, dtype=np.float64)
    T, m, batch = y.shape
    A, B = np.asarray(A, np.float64), np.asarray(B, np.float64)
    d = A.shape[0]
    m0, S0 = np.asarray(m0, np.float64), np.asarray(S0, np.float64)
    uu = np.zeros(d) if u is None else np.asarray(u, np.float64)
    tf = bool(transition_first)
    if mask is None:
        mk = np.ones((T, batch), dtype=bool)
    else:
        mk = np.asarray(mask).astype(bool)
        if mk.ndim == 1:
            mk = np.broadcast_to(mk[:, None], (T, batch)).copy()
    lp, lq = P is None, Q is None
    assert lp or lq
    Wp = np.broadcast_to(np.asarray(p_init, np.float64), (batch, d, d)).copy() if lp else None
    Wq = np.broadcast_to(np.asarray(q_init, np.float64), (batch, m, m)).copy() if lq else None
    yb = np.transpose(y, (0, 2, 1))
    hist = {k: [] for k in ("df_p", "inv_scale_p", "E_Wp", "df_q", "inv_scale_q", "E_Wq", "free_energy",
                            "free_energy_definition", "Rp_messages", "Rp_pair_form", "Rp_dense")}
    for _ in range(iterations):
        Pb = np.linalg.inv(Wp) if lp else np.asarray(P, np.float64)
        Qb = np.linalg.inv(Wq) if lq else np.asarray(Q, np.float64)
        r = lgssm.smooth_reference_schedule(y, A, B, Pb, Qb, m0, S0, mask=mk, u=u, transition_first=tf,
                                            return_messages=True)
        fe = r["neg_log_evidence"]
        qp = qq = None
        if lp:
            Pbb = np.broadcast_to(Pb, (batch, d, d))
            terms = _pair_messages(r, A, Pbb, m0, S0, uu, tf)
            Psi0 = np.asarray(p_prior[1], np.float64)
            acc = (np.full(batch, float(p_prior[0])), np.broadcast_to(Psi0, (batch, d, d)).copy())
            for Rt in terms:
                acc = R.prod_wishart(acc, (np.full(batch, d + 2.0), Rt))
            df, Psi = acc
            Rsum = terms.sum(0)
            a, b_, c_ = _wishart_block(T - 1 + int(tf), Wp, df, Psi, p_prior[0], Psi0, Rsum)
            fe = fe + a + b_ + c_
            if pair_check:
                hist["Rp_messages"].append(Rsum)
                hist["Rp_pair_form"].append(pair_form_Rp(r, A, Pbb, m0, S0, uu, tf))
                Wq_d = Wq if lq else np.broadcast_to(np.linalg.inv(Qb), (batch, m, m))
                dn = []
                for c in range(batch):
                    mu_c, Sig_c, n, _ = dense_posterior(y, mk, A, B, m0, S0, uu, tf, Wp, Wq_d, c)
                    dn.append(dense_Rp(mu_c, Sig_c, n, A, uu))
                hist["Rp_dense"].append(np.stack(dn))
            qp = (df, Psi, float(p_prior[0]), Psi0)
            Wpn = R.wishart_mean(acc)
            hist["df_p"].append(df); hist["inv_scale_p"].append(np.moveaxis(Psi, 0, 2)); hist["E_Wp"].append(np.moveaxis(Wpn, 0, 2))
        if lq:      # test_vmp_wishart.lgssm_wishart_precision's fold, operation for operation
            mu = np.transpose(r["mean"], (0, 2, 1))
            Sg = np.transpose(r["cov"], (0, 3, 1, 2))
            Psi0 = np.asarray(q_prior[1], np.float64)
            acc = (np.full(batch, float(q_prior[0])), np.broadcast_to(Psi0, (batch, m, m)).copy())
            Rsum = np.zeros((batch, m, m))
            for t in range(T):
                q_mu = (np.einsum("ij,bj->bi", B, mu[t]), B @ Sg[t] @ B.T)
                msg = R.mvnormal_meanprec_lambda((yb[t], np.zeros((batch, m, m))), q_mu)
                new = R.prod_wishart(acc, msg)
                o = mk[t]
                acc = (np.where(o, new[0], acc[0]), np.where(o[:, None, None], new[1], acc[1]))
                Rsum += np.where(o[:, None, None], msg[1], 0.0)
            df, Psi = acc
            Wqn = R.wishart_mean(acc)
            nobs = mk.sum(0)
            Elog = _mvdigamma(0.5 * df, m) + m * np.log(2.0) - np.linalg.slogdet(Psi)[1]
            fe = (fe + 0.5 * nobs * (np.linalg.slogdet(Wq)[1] - Elog)
                  + 0.5 * np.einsum("bij,bji->b", Wqn - Wq, Rsum) + wishart_kl(df, Psi, float(q_prior[0]), Psi0))
            qq = (df, Psi, float(q_prior[0]), Psi0)
            hist["df_q"].append(df); hist["inv_scale_q"].append(np.moveaxis(Psi, 0, 2)); hist["E_Wq"].append(np.moveaxis(Wqn, 0, 2))
        if definition:
            hist["free_energy_definition"].append(_free_energy_definition(
                y, mk, A, B, m0, S0, uu, tf, None if lp else Pb, None if lq else Qb, Wp, Wq, qp, qq))
        hist["free_energy"].append(fe)
        if lp:
            Wp = Wpn
        if lq:
            Wq = Wqn
    out = {k: np.stack(v) for k, v in hist.items() if v}
    out["mean"], out["cov"] = r["mean"], r["cov"]
    return out


def p_prior(d):
    return float(d + 2), np.eye(d) * 0.2


def q_prior(m):
    return float(m + 2), np.eye(m) * 0.5


def learn_kwargs(mod, learn, d, m, p_init=None, q_init=None):
    """Arguments of the reference / Context for learn = "P" or "PQ" (or "Q")."""
    kw = {}
    if "P" in learn:
        kw.update(p_prior=p_prior(d), p_init=np.linalg.inv(mod["P"]) if p_init is None else p_init)
    else:
        kw["P"] = mod["P"]
    if "Q" in learn:
        kw.update(q_prior=q_prior(m), q_init=np.eye(m) * 1.5 if q_init is None else q_init)
    else:
        kw["Q"] = np.eye(m) * 0.5
    return kw


# ====================================================================================== closed form vs definition
FE_CASES = [("P", 1, 1, False, False, None), ("P", 2, 3, True, False, "gaps"), ("P", 3, 2, False, True, "shared"),
            ("PQ", 2, 2, False, False, None), ("PQ", 2, 3, True, True, "gaps"), ("PQ", 3, 2, True, False, "shared"),
            ("PQ", 1, 2, False, True, "gaps"), ("P", 3, 3, True, True, "gaps")]


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


@pytest.mark.parametrize("learn,d,m,tf,with_u,mask", FE_CASES)
def test_closed_form_free_energy_equals_the_definition(learn, d, m, tf, with_u, mask):
    """learn-P and learn-both, several (d, m) including m > d and m < d, masks with the first and last step missing and an
    all-missing chain, transition_first and a constant u: the closed form agrees with the dense evaluation of the definition
    (transition factors' average energy under q(w_p) included) to 1e-10; the pair-form R_p equals the dense-joint R_p and
    the message-by-message R_p to 1e-10."""
    T, batch = 6, 4
    mod, y, _, _ = random_problem(d, m, T, batch, seed=20 * d + m + (7 if tf else 0))
    u = np.linspace(-0.3, 0.4, d) if with_u else None
    r = lgssm_wishart_noise(y, mod["A"], mod["B"], mod["m0"], mod["S0"], 4, mask=_mask(mask, T, batch), u=u,
                            transition_first=tf, definition=True, pair_check=True,
                            **learn_kwargs(mod, learn, d, m, p_init=np.eye(d) * 4.0))
    fe, fd = r["free_energy"], r["free_energy_definition"]
    assert np.abs(fe - fd).max() <= 1e-10 * max(1.0, np.abs(fd).max()), np.abs(fe - fd).max()
    scale = np.abs(r["Rp_dense"]).max()
    assert np.abs(r["Rp_pair_form"] - r["Rp_dense"]).max() <= 1e-10 * scale
    assert np.abs(r["Rp_messages"] - r["Rp_dense"]).max() <= 1e-10 * scale
    assert np.all(r["df_p"] == p_prior(d)[0] + T - 1 + int(tf))                # masks do not change N_p


@pytest.mark.parametrize("learn", ["P", "PQ"])
def test_single_step_without_transition_keeps_the_prior(learn):
    """T = 1 and no transition_first: there is no transition, N_p = 0, q(w_p) is the prior at every iteration and the
    process block of F vanishes (F = the definition, to 1e-10)."""
    d, m, batch = 2, 2, 3
    mod, y, _, _ = random_problem(d, m, 1, batch, seed=4)
    r = lgssm_wishart_noise(y, mod["A"], mod["B"], mod["m0"], mod["S0"], 3, definition=True,
                            **learn_kwargs(mod, learn, d, m, p_init=np.eye(d) * 3.0))
    nu, Psi0 = p_prior(d)
    assert np.all(r["df_p"] == nu)
    assert np.array_equal(r["inv_scale_p"], np.broadcast_to(Psi0[None, :, :, None], r["inv_scale_p"].shape))
    assert np.abs(r["free_energy"] - r["free_energy_definition"]).max() <= 1e-10 * max(1.0, np.abs(r["free_energy"]).max())


def test_learn_q_is_the_observation_precision_reference():
    """Learn-Q through the new reference equals test_vmp_wishart.lgssm_wishart_precision exactly."""
    from test_vmp_wishart import lgssm_wishart_precision
    d, m, T, batch = 3, 2, 9, 4
    mod, y, _, _ = random_problem(d, m, T, batch, seed=2)
    mask = _mask("gaps", T, batch)
    u = np.linspace(-0.2, 0.3, d)
    nu0, Psi0 = q_prior(m)
    a = lgssm_wishart_precision(y, mod["A"], mod["B"], mod["P"], mod["m0"], mod["S0"], nu0, Psi0, np.eye(m) * 1.5, 5,
                                mask=mask, u=u, transition_first=True)
    b = lgssm_wishart_noise(y, mod["A"], mod["B"], mod["m0"], mod["S0"], 5, P=mod["P"], q_prior=(nu0, Psi0),
                            q_init=np.eye(m) * 1.5, mask=mask, u=u, transition_first=True)
    for ka, kb in (("mean", "mean"), ("cov", "cov"), ("df", "df_q"), ("inv_scale", "inv_scale_q"), ("E_W", "E_Wq"),
                   ("free_energy", "free_energy")):
        assert np.array_equal(a[ka], b[kb]), ka


@pytest.mark.parametrize("learn", ["P", "PQ"])
def test_free_energy_is_non_increasing_over_30_iterations(learn):
    T, batch, d, m = 40, 6, 3, 2
    mod, y, _, _ = random_problem(d, m, T, batch, seed=7)
    r = lgssm_wishart_noise(y, mod["A"], mod["B"], mod["m0"], mod["S0"], 30, mask=_mask("gaps", T, batch),
                            transition_first=True, **learn_kwargs(mod, learn, d, m, p_init=np.eye(d) * 50.0,
                                                                  q_init=np.eye(m) * 1e3))
    fe = r["free_energy"]
    assert np.all(np.diff(fe, axis=0) <= 1e-9 * np.abs(fe[1:]))


def test_posterior_mean_recovers_the_true_process_precision():
    """T = 2000 draws with a known process precision w_p and a small known observation noise (Q = 1e-3 I, B = I): the
    states are nearly observed, so R_p / N_p is close to the sample covariance of the N_p process-noise draws, whose
    relative spread is about sqrt(2 / N_p).  E[w_p] under the final q(w_p) is within 5 sqrt(2 / T) (relative Frobenius)."""
    T, batch, d = 2000, 3, 2
    rng = np.random.default_rng(31)
    A = np.array([[0.9, 0.2], [-0.2, 0.9]])
    w_true = np.array([[4.0, 1.0], [1.0, 2.5]])
    LP = np.linalg.cholesky(np.linalg.inv(w_true))
    Q = 1e-3 * np.eye(d)
    y = np.zeros((T, d, batch))
    for c in range(batch):
        x = rng.standard_normal(d)
        for t in range(T):
            if t > 0:
                x = A @ x + LP @ rng.standard_normal(d)
            y[t, :, c] = x + np.sqrt(1e-3) * rng.standard_normal(d)
    r = lgssm_wishart_noise(y, A, np.eye(d), np.zeros(d), np.eye(d), 10, Q=Q, p_prior=p_prior(d), p_init=np.eye(d))
    for c in range(batch):
        Ew = r["E_Wp"][-1][:, :, c]
        assert np.linalg.norm(Ew - w_true) / np.linalg.norm(w_true) < 5 * np.sqrt(2.0 / T)


# ====================================================================================== argument handling (no device)
def _bare_context():
    from rxinfer_jl_b200.context import Context
    return object.__new__(Context)


def test_context_argument_rules(rx):
    c = _bare_context()
    mod, y, _, _ = random_problem(2, 2, 5, 3, seed=1)
    y = torch.as_tensor(y)
    args = (mod["A"], mod["B"], mod["m0"], mod["S0"])
    pp, qp = (4.0, np.eye(2)), (4.0, np.eye(2))
    with pytest.raises(ValueError, match="both known"):
        c.lgssm_vmp_noise(y, *args, P=mod["P"], Q=np.eye(2))
    with pytest.raises(ValueError, match="P is learned: pass p_prior"):
        c.lgssm_vmp_noise(y, *args, Q=np.eye(2), p_prior=pp)                       # no initial q(w_p)
    with pytest.raises(ValueError, match="Q is learned: pass q_prior"):
        c.lgssm_vmp_noise(y, *args, P=mod["P"], q_init=np.eye(2))
    with pytest.raises(ValueError, match="P is known"):
        c.lgssm_vmp_noise(y, *args, P=mod["P"], p_prior=pp, p_init=np.eye(2), q_prior=qp, q_init=np.eye(2))
    with pytest.raises(ValueError, match="iterations must be >= 1"):
        c.lgssm_vmp_noise(y, *args, Q=np.eye(2), p_prior=pp, p_init=np.eye(2), iterations=0)
    with pytest.raises(ValueError, match="expected \\[T, m, batch\\]"):
        c.lgssm_vmp_noise(y[0], *args, Q=np.eye(2), p_prior=pp, p_init=np.eye(2))
    with pytest.raises(ValueError, match="inv_scale_p0: expected shape"):
        c.lgssm_vmp_noise(y, *args, Q=np.eye(2), p_prior=(4.0, np.eye(3)), p_init=np.eye(2))
    with pytest.raises(ValueError, match="init_E_Wq: expected shape"):
        c.lgssm_vmp_noise(y, *args, P=mod["P"], q_prior=qp, q_init=np.eye(1))
    with pytest.raises(ValueError, match="Q: expected shape"):
        c.lgssm_vmp_noise(y, *args, Q=np.eye(3), p_prior=pp, p_init=np.eye(2))
    with pytest.raises(ValueError, match="u: expected shape"):
        c.lgssm_vmp_noise(y, *args, Q=np.eye(2), p_prior=pp, p_init=np.eye(2), u=np.ones(3))
    c.device = 0
    with pytest.raises(ValueError, match="y: expected a tensor on cuda"):
        c.lgssm_vmp_noise(y, *args, Q=np.eye(2), p_prior=pp, p_init=np.eye(2))     # data arrays are device arrays


def _noise_model(rx, **kw):
    from rxinfer_jl_b200 import inference as I
    from rxinfer_jl_b200.distributions import Wishart
    mod, _, _, _ = random_problem(2, 2, 5, 3, seed=1)
    base = dict(A=mod["A"], B=mod["B"], x0=(mod["m0"], mod["S0"]), Q=np.eye(2), p_prior=Wishart(4, np.eye(2)),
                p_init=Wishart(4, np.eye(2)))
    base.update(kw)
    return I.linear_gaussian_ssm_wishart_noise(**base)


def test_infer_argument_rules(rx):
    from rxinfer_jl_b200 import inference as I
    model = _noise_model(rx)
    y = torch.zeros(5, 2, 3)
    with pytest.raises(NotImplementedError, match="input sequences"):
        I.infer(model=model, data={"y": y, "u": np.zeros((5, 2))}, iterations=3)
    with pytest.raises(NotImplementedError, match="predictions"):
        I.infer(model=model, data={"y": y}, iterations=3, predictvars={"y": I.KeepLast()})
    with pytest.raises(NotImplementedError, match="KeepLast"):
        I.infer(model=model, data={"y": y}, iterations=3, returnvars={"x": I.KeepEach()})
    with pytest.raises(ValueError, match="needs `data`"):
        I.infer(model=model, iterations=3)


def _shim():
    import os
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    return open(os.path.join(root, "rxinfer.jl_b200", "julia", "RxGaussB200.jl")).read()


def test_julia_helper_packs_the_call():
    """`lgssm_wishart_noise(ctx, y; ...)` refuses a missing initial q(w) and two known noises, passes row-major host
    matrices, NULL for what a known noise does not have, and an fp64 free-energy buffer to the export."""
    s = _shim()
    body = s[s.index("function lgssm_wishart_noise(ctx::Context"):]
    body = body[:body.index("\nend\n")]
    assert "batch, m, T = size(y)" in body
    assert "is learned: pass its prior" in body and "both known" in body
    assert "permutedims" in body and "Lib.lgssm_vmp_noise(ctx, d, m, T, batch, iterations" in body
    assert "ptr(Pt), nup, ptr(iSp0), ptr(EWp0), ptr(Qt), nuq, ptr(iSq0), ptr(EWq0)" in body
    assert "reinterpret(Float64" in body and "RXG_TRANSITION_FIRST" in body
