"""fp64 reference of the Wishart-precision VMP around the LGSSM smoother (rxg_lgssm_vmp_wishart_f32), and its CPU checks.

Model (per chain): w ~ Wishart(nu0, inv(Psi0)); x[1] ~ N(m0, S0) (or one transition earlier); x[t] ~ N(A x[t-1] + u, P);
y[t] ~ N(B x[t], inv(w)); q(x) q(w).  ``lgssm_wishart_precision`` runs the schedule message by message:
  q(x)  oracle.lgssm.smooth_reference_schedule with the per-chain Q = inv(E[w]) of the previous q(w);
  q(w)  the prior folded with MvNormalMeanPrecision(:Lambda)(q_out = PointMass(y_t), q_mu = N(B mu_t, B Sigma_t B')) messages
        (oracle.rules.mvnormal_meanprec_lambda / prod_wishart), one per observed step;
  F     the Bethe free energy in closed form (what the kernel evaluates) and, with ``definition=True``, from its definition
        E_q[-log p(y, x, w)] - H[q(x)] - H[q(w)] with a dense (T d)-dimensional Gaussian q(x).
"""
import numpy as np
import pytest
import torch
from scipy.special import digamma, gammaln

from oracle import lgssm, rules as R
from oracle import vmp as oracle_vmp


def _mvlgamma(a, m):
    return m * (m - 1) / 4.0 * np.log(np.pi) + sum(gammaln(a - 0.5 * i) for i in range(m))


def _mvdigamma(a, m):
    return sum(digamma(a - 0.5 * i) for i in range(m))


def wishart_kl(df, Psi, nu0, Psi0):
    """KL(Wishart(df, inv(Psi)) || Wishart(nu0, inv(Psi0))), inverse scales Psi[batch, m, m] / Psi0[m, m]."""
    m = Psi.shape[-1]
    Pinv = np.linalg.inv(Psi)
    ld = np.linalg.slogdet(Psi)[1]
    ld0 = np.linalg.slogdet(Psi0)[1]
    trP = np.einsum("ij,bji->b", Psi0, Pinv)
    return (-0.5 * nu0 * (ld0 - ld) + 0.5 * df * (trP - m) + _mvlgamma(0.5 * nu0, m) - _mvlgamma(0.5 * df, m)
            + 0.5 * (df - nu0) * _mvdigamma(0.5 * df, m))


def _dense_prior(A, P, m0, S0, u, T, transition_first):
    """Information form (J0, h0) of the Gaussian chain prior over X = (x_1, ..., x_T)."""
    d = A.shape[0]
    u = np.zeros(d) if u is None else np.asarray(u, np.float64)
    if transition_first:
        m1, S1 = A @ m0 + u, A @ S0 @ A.T + P
    else:
        m1, S1 = np.asarray(m0, np.float64), np.asarray(S0, np.float64)
    J0 = np.zeros((T * d, T * d)); h0 = np.zeros(T * d)
    L1 = np.linalg.inv(S1)
    J0[:d, :d] += L1; h0[:d] += L1 @ m1
    Pi = np.linalg.inv(P)
    for t in range(1, T):
        a, c = slice((t - 1) * d, t * d), slice(t * d, (t + 1) * d)
        J0[c, c] += Pi; J0[a, a] += A.T @ Pi @ A
        J0[c, a] -= Pi @ A; J0[a, c] -= A.T @ Pi
        h0[c] += Pi @ u; h0[a] -= A.T @ Pi @ u
    return J0, h0


def _free_energy_definition(y, mk, A, B, P, m0, S0, u, tf, Wbar, df, Psi, nu0, Psi0):
    """F = E_q[-log p(x)] + E_q[-log p(y | x, w)] + E_q[-log p(w)] - H[q(x)] - H[q(w)], q(x) the exact posterior
    under N(y | Bx, inv(Wbar)), one chain at a time with dense algebra."""
    T, m, batch = y.shape
    d = A.shape[0]
    J0, h0 = _dense_prior(A, P, m0, S0, u, T, tf)
    mu0 = np.linalg.solve(J0, h0)
    ld_J0 = np.linalg.slogdet(J0)[1]
    out = np.zeros(batch)
    for c in range(batch):
        J, h = J0.copy(), h0.copy()
        for t in range(T):
            if mk[t, c]:
                s = slice(t * d, (t + 1) * d)
                J[s, s] += B.T @ Wbar[c] @ B
                h[s] += B.T @ Wbar[c] @ y[t, :, c]
        Sig = np.linalg.inv(J); mu = Sig @ h
        dm = mu - mu0
        E_px = 0.5 * (T * d * np.log(2 * np.pi) - ld_J0 + np.trace(J0 @ Sig) + dm @ J0 @ dm)
        H_x = 0.5 * (T * d * (1 + np.log(2 * np.pi)) + np.linalg.slogdet(Sig)[1])
        Ew = df[c] * np.linalg.inv(Psi[c])
        ld_S = -np.linalg.slogdet(Psi[c])[1]                       # log det of the scale inv(Psi)
        Elog = _mvdigamma(0.5 * df[c], m) + m * np.log(2.0) + ld_S
        E_py = 0.0
        for t in range(T):
            if mk[t, c]:
                s = slice(t * d, (t + 1) * d)
                e = y[t, :, c] - B @ mu[s]
                Rt = np.outer(e, e) + B @ Sig[s, s] @ B.T
                E_py += 0.5 * (m * np.log(2 * np.pi) - Elog + np.trace(Ew @ Rt))
        E_pw = (-0.5 * (nu0 - m - 1) * Elog + 0.5 * np.trace(Psi0 @ Ew) + 0.5 * nu0 * m * np.log(2.0)
                - 0.5 * nu0 * np.linalg.slogdet(Psi0)[1] + _mvlgamma(0.5 * nu0, m))
        H_w = (0.5 * df[c] * ld_S + 0.5 * df[c] * m * np.log(2.0) + _mvlgamma(0.5 * df[c], m)
               - 0.5 * (df[c] - m - 1) * Elog + 0.5 * df[c] * m)
        out[c] = E_px + E_py + E_pw - H_x - H_w
    return out


def lgssm_wishart_precision(y, A, B, P, m0, S0, nu0, inv_scale0, init_E_W, iterations, mask=None, u=None,
                            transition_first=False, definition=False):
    """y[T, m, batch] (fp64 or the fp32 values the device sees); mask None, [T, batch] or a shared [T] pattern.
    Returns dict(mean[T, d, batch], cov[T, d, d, batch] of the last iteration, df[iterations, batch],
    inv_scale[iterations, m, m, batch], E_W[iterations, m, m, batch], free_energy[iterations, batch] (closed form) and, with
    ``definition``, free_energy_definition[iterations, batch])."""
    y = np.asarray(y, dtype=np.float64)
    T, m, batch = y.shape
    A, B, P = (np.asarray(M, np.float64) for M in (A, B, P))
    m0, S0 = np.asarray(m0, np.float64), np.asarray(S0, np.float64)
    Psi0 = np.asarray(inv_scale0, np.float64)
    if mask is None:
        mk = np.ones((T, batch), dtype=bool)
    else:
        mk = np.asarray(mask).astype(bool)
        if mk.ndim == 1:
            mk = np.broadcast_to(mk[:, None], (T, batch)).copy()
    W = np.broadcast_to(np.asarray(init_E_W, np.float64), (batch, m, m)).copy()
    yb = np.transpose(y, (0, 2, 1))                                    # [T, batch, m]
    hist = dict(df=[], inv_scale=[], E_W=[], free_energy=[], free_energy_definition=[])
    for _ in range(iterations):
        Q = np.linalg.inv(W)
        r = lgssm.smooth_reference_schedule(y, A, B, P, Q, m0, S0, mask=mk, u=u, transition_first=transition_first)
        mu = np.transpose(r["mean"], (0, 2, 1))                        # [T, batch, d]
        Sg = np.transpose(r["cov"], (0, 3, 1, 2))                      # [T, batch, d, d]
        acc = (np.full(batch, float(nu0)), np.broadcast_to(Psi0, (batch, m, m)).copy())
        Rsum = np.zeros((batch, m, m))
        for t in range(T):
            q_mu = (np.einsum("ij,bj->bi", B, mu[t]), B @ Sg[t] @ B.T)
            msg = R.mvnormal_meanprec_lambda((yb[t], np.zeros((batch, m, m))), q_mu)
            new = R.prod_wishart(acc, msg)
            o = mk[t]
            acc = (np.where(o, new[0], acc[0]), np.where(o[:, None, None], new[1], acc[1]))
            Rsum += np.where(o[:, None, None], msg[1], 0.0)
        df, Psi = acc
        Wn = R.wishart_mean(acc)
        nobs = mk.sum(0)
        Elog = _mvdigamma(0.5 * df, m) + m * np.log(2.0) - np.linalg.slogdet(Psi)[1]
        fe = (r["neg_log_evidence"] + 0.5 * nobs * (np.linalg.slogdet(W)[1] - Elog)
              + 0.5 * np.einsum("bij,bji->b", Wn - W, Rsum) + wishart_kl(df, Psi, float(nu0), Psi0))
        if definition:
            hist["free_energy_definition"].append(_free_energy_definition(y, mk, A, B, P, m0, S0, u, transition_first, W,
                                                                          df, Psi, float(nu0), Psi0))
        hist["df"].append(df); hist["inv_scale"].append(np.moveaxis(Psi, 0, 2)); hist["E_W"].append(np.moveaxis(Wn, 0, 2))
        hist["free_energy"].append(fe)
        W = Wn
    out = {k: np.stack(v) for k, v in hist.items() if v}
    out["mean"], out["cov"] = r["mean"], r["cov"]
    return out


def random_problem(d, m, T, batch, seed, w_true=None):
    """A stable random model and data drawn from it with a per-chain observation precision w (default: a random SPD
    matrix per chain); y is rounded to fp32 once, as the device sees it."""
    rng = np.random.default_rng(seed)
    Qr, _ = np.linalg.qr(rng.standard_normal((d, d)))
    A = 0.95 * Qr
    B = rng.standard_normal((m, d)) / np.sqrt(d)
    G = rng.standard_normal((d, d)) * 0.2
    P = 0.1 * np.eye(d) + G @ G.T * 0.1
    m0 = rng.standard_normal(d) * 0.5
    S0 = np.eye(d) * 2.0
    ws = []
    x = np.zeros((T, d, batch)); y = np.zeros((T, m, batch))
    for b in range(batch):
        if w_true is None:
            H = rng.standard_normal((m, m)) * 0.4
            w = np.eye(m) * 2.0 + H @ H.T
        else:
            w = np.asarray(w_true, np.float64)
        ws.append(w)
        Lw = np.linalg.cholesky(np.linalg.inv(w)); LP = np.linalg.cholesky(P)
        xt = m0 + np.linalg.cholesky(S0) @ rng.standard_normal(d)
        for t in range(T):
            if t > 0:
                xt = A @ xt + LP @ rng.standard_normal(d)
            x[t, :, b] = xt
            y[t, :, b] = B @ xt + Lw @ rng.standard_normal(m)
    f32 = lambda M: np.asarray(M, np.float32).astype(np.float64)
    return dict(A=f32(A), B=f32(B), P=f32(P), m0=f32(m0), S0=f32(S0)), y.astype(np.float32), np.stack(ws), x


def w_prior(m):
    return float(m + 2), np.eye(m) * 0.5


# ====================================================================================== closed form vs definition
FE_CASES = [(1, 1, False, False, None), (2, 2, False, False, None), (2, 3, True, False, "gaps"), (3, 2, False, True, "gaps"),
            (1, 2, True, True, "shared"), (3, 3, True, True, "gaps")]


def _mask(kind, T, batch):
    if kind is None:
        return None
    if kind == "shared":
        mk = np.ones(T, dtype=np.uint8); mk[0] = 0; mk[-1] = 0
        return mk
    mk = np.ones((T, batch), dtype=np.uint8)
    mk[0, 0] = 0; mk[-1, 1] = 0; mk[2:4, 2] = 0
    mk[:, -1] = 0                                         # a chain with N_b = 0
    return mk


@pytest.mark.parametrize("d,m,tf,with_u,mask", FE_CASES)
def test_closed_form_free_energy_equals_the_definition(d, m, tf, with_u, mask):
    """Several (d, m) including m > d, masks with the first and last step missing and a chain with N_b = 0,
    transition_first and a constant u: the closed form agrees with the dense evaluation of the definition to 1e-10."""
    T, batch = 6, 4
    mod, y, _, _ = random_problem(d, m, T, batch, seed=10 * d + m)
    u = np.linspace(-0.3, 0.4, d) if with_u else None
    nu0, Psi0 = w_prior(m)
    r = lgssm_wishart_precision(y, mod["A"], mod["B"], mod["P"], mod["m0"], mod["S0"], nu0, Psi0, np.eye(m) * 1.5, 4,
                                mask=_mask(mask, T, batch), u=u, transition_first=tf, definition=True)
    fe, fd = r["free_energy"], r["free_energy_definition"]
    assert np.abs(fe - fd).max() <= 1e-10 * max(1.0, np.abs(fd).max()), np.abs(fe - fd).max()
    if mask is not None and mask != "shared":
        assert np.all(r["df"][:, -1] == nu0) and np.allclose(fe[:, -1], 0.0, atol=1e-12)     # N_b = 0: q(w) = prior, F = 0


def test_scalar_case_is_the_gamma_precision_oracle():
    """At d = m = 1, Wishart(nu, Psi) is Gamma(nu / 2, Psi / 2): with nu0 = 2 a0, Psi0 = 2 b0 the reference reproduces
    oracle.vmp.lgssm_gamma_precision (df = 2 shape, Psi = 2 rate, same posteriors and free energy) to 1e-12."""
    T, batch, its = 12, 5, 6
    rng = np.random.default_rng(3)
    y = np.cumsum(rng.standard_normal((T, batch)), axis=0) + rng.standard_normal((T, batch)) * 0.7
    a, v, prior, (a0, b0), Etau = 0.9, 0.5, (0.3, 4.0), (1.5, 2.0), 0.8
    g = oracle_vmp.lgssm_gamma_precision(y, A_scalar=a, prior=prior, proc_var=v, gamma_prior=(a0, b0), iterations=its,
                                         init_Etau=Etau, return_free_energy=True)
    r = lgssm_wishart_precision(y[:, None, :], [[a]], [[1.0]], [[v]], [prior[0]], [[prior[1]]], 2 * a0, [[2 * b0]],
                                [[Etau]], its)
    assert np.allclose(r["df"][-1], 2 * g["shape"], rtol=0, atol=1e-12)
    assert np.allclose(r["inv_scale"][-1, 0, 0], 2 * g["rate"], rtol=1e-12, atol=0)
    assert np.allclose(r["mean"][:, 0], g["mean"], rtol=1e-12, atol=1e-12)
    assert np.allclose(r["cov"][:, 0, 0], g["var"], rtol=1e-12, atol=0)
    assert np.allclose(r["free_energy"], g["free_energy"], rtol=1e-12, atol=1e-10)


def test_free_energy_is_non_increasing_over_30_iterations():
    T, batch = 40, 6
    mod, y, _, _ = random_problem(3, 2, T, batch, seed=7)
    nu0, Psi0 = w_prior(2)
    r = lgssm_wishart_precision(y, mod["A"], mod["B"], mod["P"], mod["m0"], mod["S0"], nu0, Psi0, np.eye(2) * 1e3, 30,
                                mask=_mask("gaps", T, batch))
    fe = r["free_energy"]
    assert np.all(np.diff(fe, axis=0) <= 1e-9 * np.abs(fe[1:]))


def test_posterior_mean_recovers_the_true_precision():
    """T = 2000 draws from the model with a known w: E[w] under the final q(w) is within 5 sqrt(2 / T) (relative
    Frobenius; the sampling spread of a precision estimate from T residuals is about sqrt(2 / T)) of the truth."""
    T, batch = 2000, 3
    w_true = np.array([[2.0, 0.6], [0.6, 1.0]])
    mod, y, _, _ = random_problem(2, 2, T, batch, seed=11, w_true=w_true)
    nu0, Psi0 = w_prior(2)
    r = lgssm_wishart_precision(y, mod["A"], mod["B"], mod["P"], mod["m0"], mod["S0"], nu0, Psi0, np.eye(2), 15)
    for c in range(batch):
        Ew = r["E_W"][-1][:, :, c]
        assert np.linalg.norm(Ew - w_true) / np.linalg.norm(w_true) < 5 * np.sqrt(2.0 / T)


# ====================================================================================== argument handling (no device)
def _bare_context():
    from rxinfer_jl_b200.context import Context
    return object.__new__(Context)


def test_context_argument_rules(rx):
    c = _bare_context()
    mod, y, _, _ = random_problem(2, 2, 5, 3, seed=1)
    y = torch.as_tensor(y)
    args = (mod["A"], mod["B"], mod["P"], mod["m0"], mod["S0"])
    with pytest.raises(ValueError, match="iterations must be >= 1"):
        c.lgssm_vmp_wishart(y, *args, iterations=0)
    with pytest.raises(ValueError, match="expected \\[T, m, batch\\]"):
        c.lgssm_vmp_wishart(y[0], *args)
    with pytest.raises(ValueError, match="inv_scale0: expected shape"):
        c.lgssm_vmp_wishart(y, *args, w_prior=(3.0, np.eye(3)))
    with pytest.raises(ValueError, match="init_E_W: expected shape"):
        c.lgssm_vmp_wishart(y, *args, init_E_W=np.eye(1))
    with pytest.raises(ValueError, match="u: expected shape"):
        c.lgssm_vmp_wishart(y, *args, u=np.ones(3))
    c.device = 0
    with pytest.raises(ValueError, match="y: expected a tensor on cuda"):
        c.lgssm_vmp_wishart(y, *args)                        # data arrays are device arrays


def _wishart_model(rx, **kw):
    from rxinfer_jl_b200 import inference as I
    from rxinfer_jl_b200.distributions import Wishart
    mod, _, _, _ = random_problem(2, 2, 5, 3, seed=1)
    return I.linear_gaussian_ssm_wishart_precision(A=mod["A"], B=mod["B"], P=mod["P"], x0=(mod["m0"], mod["S0"]),
                                                   w_prior=Wishart(3, np.eye(2)), w_init=Wishart(2, 1e12 * np.eye(2)), **kw)


def test_infer_argument_rules(rx):
    from rxinfer_jl_b200 import inference as I
    model = _wishart_model(rx)
    y = torch.zeros(5, 2, 3)
    with pytest.raises(NotImplementedError, match="input sequences"):
        I.infer(model=model, data={"y": y, "u": np.zeros((5, 2))}, iterations=3)
    with pytest.raises(NotImplementedError, match="predictions"):
        I.infer(model=model, data={"y": y}, iterations=3, predictvars={"y": I.KeepLast()})
    with pytest.raises(NotImplementedError, match="KeepLast"):
        I.infer(model=model, data={"y": y}, iterations=3, returnvars={"x": I.KeepEach()})
    with pytest.raises(ValueError, match="needs `data`"):
        I.infer(model=model, iterations=3)


def test_wishart_conversion():
    from rxinfer_jl_b200.distributions import Wishart
    S = np.array([[2.0, 0.5], [0.5, 1.0]])
    w = Wishart(5, S)
    assert np.allclose(w.inv_scale() @ S, np.eye(2)) and np.allclose(w.mean(), 5 * S)


def _shim():
    import os
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    return open(os.path.join(root, "rxinfer.jl_b200", "julia", "RxGaussB200.jl")).read()


def test_julia_helper_packs_the_call():
    """`lgssm_wishart(ctx, y; ...)` passes row-major host matrices, the prior's (df, inverse scale), the vague default of
    the initial E[w] and an fp64 free-energy buffer to the export."""
    s = _shim()
    body = s[s.index("function lgssm_wishart(ctx::Context"):]
    body = body[:body.index("\nend\n")]
    assert "batch, m, T = size(y)" in body
    assert "Matrix{Float32}(m * 1f12 * I, m, m)" in body                  # mean of vague(Wishart, m)
    assert "permutedims" in body and "Lib.lgssm_vmp_wishart(ctx, d, m, T, batch, iterations" in body
    assert "reinterpret(Float64" in body and "RXG_TRANSITION_FIRST" in body
