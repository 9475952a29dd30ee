"""Known per-step inputs (control / exogenous terms) of the batched LGSSM sweeps: x[t] ~ N(A x[t-1] + u[t], P).

CPU half: the fp64 references the GPU tests gate against, checked against the oracle and against each other, and the
argument handling of ``Context`` and ``infer``.

Two references, both fp64 and independent of the library:
  * ``input_mean_side``: the gain-table form (chain-independent covariance side of ``test_shared_sweep_variants``, mean
    recursion with u[t]), batched over chains in torch;
  * ``kalman_rts_inputs``: a textbook Kalman filter + RTS smoother batched over chains with per-chain models, per-chain
    masks and per-chain inputs (every covariance per chain).
Row t of the sequence enters the transition into x[t]; row 0 is used only with ``transition_first``.
"""
import numpy as np
import pytest
import torch

from oracle import lgssm
from test_shared_sweep_variants import LOG2PI, covariance_side, random_model, reference_sweep, simulate


# ====================================================================================== references
def _seq(u, T, d, nb, dev):
    """u[T, d] (shared) or u[T, d, batch] (per chain) -> fp64 [T, d, batch] (a view for the shared form)."""
    u = torch.as_tensor(np.asarray(u) if not isinstance(u, torch.Tensor) else u).to(dev, torch.float64)
    return u[..., None].expand(u.shape[0], d, nb) if u.dim() == 2 else u


def input_mean_side(cs, mod, y, useq, *, smooth=True, mu0=None):
    """Mean recursion of a shared model with inputs: (mean[T, d, batch], nle[batch]) in fp64 on y's device."""
    dev = y.device
    T, m, nb = y.shape
    t64 = lambda a: torch.as_tensor(np.asarray(a, np.float64), dtype=torch.float64, device=dev)
    A, B = t64(mod["A"]), t64(mod["B"])
    d = A.shape[0]
    U = _seq(useq, T, d, nb, dev)
    K, G, Si, half = t64(cs["K"]), t64(cs["G"]), t64(cs["Sinv"]), cs["half"]
    tf = cs["transition_first"]
    mu = (mu0.to(dev, torch.float64) if mu0 is not None else t64(mod["m0"]).reshape(d, 1).expand(d, nb)).clone()
    mean = torch.empty(T, d, nb, dtype=torch.float64, device=dev)
    nle = torch.zeros(nb, dtype=torch.float64, device=dev)
    for t in range(T):
        if t > 0 or tf:
            mu = A @ mu + U[t]
        if cs["obs"][t]:
            e = y[t].to(torch.float64) - B @ mu
            nle += half[t] + 0.5 * (e * (Si[t] @ e)).sum(0)
            mu = mu + K[t] @ e
        mean[t] = mu
    if smooth:
        for t in range(T - 2, -1, -1):
            mean[t] += G[t] @ (mean[t + 1] - (A @ mean[t] + U[t + 1]))
    return mean, nle


def input_reference(mod, y, useq, *, smooth=True, transition_first=False, tmask=None, mu0=None, cs=None):
    """dict(mean[T, d, batch], cov[T, d, d], nle[batch]) of a shared model with inputs (shared or per-chain sequence)."""
    cs = cs if cs is not None else covariance_side(mod, y.shape[0], tmask, transition_first)
    mean, nle = input_mean_side(cs, mod, y, useq, smooth=smooth, mu0=mu0)
    return dict(mean=mean, cov=cs["Ss"] if smooth else cs["Sf"], nle=nle)


def kalman_rts_inputs(mods, y, useq, *, mask=None, smooth=True, transition_first=False):
    """Textbook Kalman filter + RTS smoother of every chain, fp64, batched over chains.

    ``mods``: dict of per-chain model arrays A[b, d, d], B[b, m, d], P, Q, m0[b, d], S0 (torch fp64, any device);
    ``useq``: [T, d] or [T, d, batch]; ``mask[T, batch]`` (1 = observed) or None.
    Returns dict(mean[T, d, batch], cov[T, d, d, batch], nle[batch])."""
    A, B, P, Q, m0, S0 = (mods[k] for k in ("A", "B", "P", "Q", "m0", "S0"))
    dev = A.device
    T, m, nb = y.shape
    d = A.shape[-1]
    U = _seq(useq, T, d, nb, dev).permute(0, 2, 1)          # [T, b, d]
    Y = y.to(dev, torch.float64).permute(0, 2, 1)            # [T, b, m]
    obs = torch.ones(T, nb, dtype=torch.bool, device=dev) if mask is None else torch.as_tensor(mask, device=dev).bool()
    At, Bt = A.transpose(-1, -2), B.transpose(-1, -2)
    mu, S = m0.clone(), S0.clone()
    fm = torch.empty(T, nb, d, dtype=torch.float64, device=dev); fS = torch.empty(T, nb, d, d, dtype=torch.float64, device=dev)
    pS = torch.empty_like(fS)
    nle = torch.zeros(nb, dtype=torch.float64, device=dev)
    for t in range(T):
        if t > 0 or transition_first:
            mu = (A @ mu[..., None])[..., 0] + U[t]
            S = A @ S @ At + P
        pS[t] = S
        Sn = B @ S @ Bt + Q
        e = Y[t] - (B @ mu[..., None])[..., 0]
        Ki = torch.linalg.solve(Sn, B @ S).transpose(-1, -2)      # S B' Sn^-1
        q = (e[..., None].transpose(-1, -2) @ torch.linalg.solve(Sn, e[..., None]))[..., 0, 0]
        o = obs[t]
        nle += torch.where(o, 0.5 * (m * LOG2PI + torch.linalg.slogdet(Sn)[1] + q), torch.zeros_like(q))
        mu = torch.where(o[:, None], mu + (Ki @ e[..., None])[..., 0], mu)
        S = torch.where(o[:, None, None], S - Ki @ Sn @ Ki.transpose(-1, -2), S)
        S = 0.5 * (S + S.transpose(-1, -2))
        fm[t], fS[t] = mu, S
    if smooth:
        sm, sS = fm.clone(), fS.clone()
        for t in range(T - 2, -1, -1):
            G = torch.linalg.solve(pS[t + 1], A @ fS[t]).transpose(-1, -2)     # fS A' pS^-1
            sm[t] = fm[t] + (G @ (sm[t + 1] - (A @ fm[t][..., None])[..., 0] - U[t + 1])[..., None])[..., 0]
            sS[t] = fS[t] + G @ (sS[t + 1] - pS[t + 1]) @ G.transpose(-1, -2)
        fm, fS = sm, sS
    return dict(mean=fm.permute(0, 2, 1), cov=fS.permute(0, 2, 3, 1), nle=nle)


def per_chain_models(mod, nb, dev="cpu"):
    """The shared model replicated per chain ([b, ...] fp64 torch)."""
    t = lambda k, s: torch.as_tensor(np.asarray(mod[k], np.float64), device=dev).expand(nb, *s).clone()
    d, m = mod["A"].shape[0], mod["B"].shape[0]
    return dict(A=t("A", (d, d)), B=t("B", (m, d)), P=t("P", (d, d)), Q=t("Q", (m, m)), m0=t("m0", (d,)), S0=t("S0", (d, d)))


def input_sequence(T, d, seed, nb=None):
    """A random input sequence: [T, d] (shared), or [T, d, nb] (per chain) fp32."""
    rng = np.random.default_rng(seed)
    shape = (T, d) if nb is None else (T, d, nb)
    return (0.7 * rng.standard_normal(shape)).astype(np.float32)


def _rel(a, b):
    a = np.asarray(a, np.float64); b = np.asarray(b, np.float64)
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-300))


# ====================================================================================== CPU: the references
CASES = [(1, 1), (2, 1), (4, 4), (3, 2), (6, 6)]


@pytest.mark.parametrize("d,m", CASES)
@pytest.mark.parametrize("tf", [False, True])
@pytest.mark.parametrize("per_chain", [False, True])
@pytest.mark.parametrize("masked", [False, True])
def test_gain_form_matches_textbook_with_inputs(d, m, tf, per_chain, masked):
    """The gain-table form with u[t] = the textbook Kalman + RTS smoother with u[t] (1e-10), for a shared and a per-chain
    sequence, with a shared missing-data pattern."""
    mod = random_model(d, m, seed=10 * d + m)
    T, nb = 23, 5
    y = torch.as_tensor(simulate(mod, T, nb, seed=d + m))
    useq = input_sequence(T, d, seed=d * m + 1, nb=nb if per_chain else None)
    tm = None
    if masked:
        tm = np.ones(T, np.uint8); tm[0] = 0; tm[7:12] = 0; tm[-1] = 0
    for smooth in (True, False):
        g = input_reference(mod, y, useq, smooth=smooth, transition_first=tf, tmask=tm)
        full = None if tm is None else np.repeat(tm[:, None], nb, axis=1)
        k = kalman_rts_inputs(per_chain_models(mod, nb), y, useq, mask=full, smooth=smooth, transition_first=tf)
        assert _rel(g["mean"].numpy(), k["mean"].numpy()) < 1e-10
        assert _rel(np.broadcast_to(g["cov"][..., None], k["cov"].shape), k["cov"].numpy()) < 1e-10
        assert np.allclose(g["nle"].numpy(), k["nle"].numpy(), rtol=1e-10, atol=1e-10)


@pytest.mark.parametrize("d,m", CASES)
@pytest.mark.parametrize("tf", [False, True])
def test_constant_sequence_is_the_constant_offset(d, m, tf):
    """A sequence whose rows are all u gives the oracle's constant-u smoother; an all-zero sequence gives the oracle
    without an offset (1e-10)."""
    mod = random_model(d, m, seed=20 + 10 * d + m)
    T, nb = 19, 4
    y = simulate(mod, T, nb, seed=3 * d + m)
    u = (0.5 * np.random.default_rng(d).standard_normal(d))
    for uu, useq in ((u, np.tile(u, (T, 1))), (None, np.zeros((T, d)))):
        ora = lgssm.smooth_reference_schedule(y, **mod, u=uu, transition_first=tf)
        k = kalman_rts_inputs(per_chain_models(mod, nb), torch.as_tensor(y), useq, transition_first=tf)
        g = input_reference(mod, torch.as_tensor(y), useq, transition_first=tf)
        for ref in (k, g):
            assert _rel(ref["mean"].numpy(), ora["mean"]) < 1e-10
            assert np.allclose(ref["nle"].numpy(), ora["neg_log_evidence"], rtol=1e-10, atol=1e-10)
        assert _rel(k["cov"].numpy(), ora["cov"]) < 1e-10


@pytest.mark.parametrize("d,m", CASES)
@pytest.mark.parametrize("tf", [False, True])
def test_linearity_identity(d, m, tf):
    """E[x | y, u] = z + E[xi | y - B z] with z_t = A z_{t-1} + u_t (z = 0 at the prior): the route of the large-state
    family.  The evidence is the same (the shift has a Jacobian of 1), and so are the covariances."""
    mod = random_model(d, m, seed=40 + 10 * d + m)
    T, nb = 17, 6
    y = simulate(mod, T, nb, seed=5 * d + m).astype(np.float64)
    useq = input_sequence(T, d, seed=7, nb=nb).astype(np.float64)
    A, B = mod["A"].astype(np.float64), mod["B"].astype(np.float64)
    z = np.zeros((T, d, nb)); zc = np.zeros((d, nb))
    for t in range(T):
        if t > 0 or tf:
            zc = A @ zc + useq[t]
        z[t] = zc
    ys = y - np.einsum("kd,tdb->tkb", B, z)
    xi = lgssm.smooth_reference_schedule(ys, **mod, transition_first=tf)
    k = kalman_rts_inputs(per_chain_models(mod, nb), torch.as_tensor(y), useq, transition_first=tf)
    assert _rel(z + xi["mean"], k["mean"].numpy()) < 1e-10
    assert np.allclose(xi["neg_log_evidence"], k["nle"].numpy(), rtol=1e-10, atol=1e-10)
    assert _rel(xi["cov"], k["cov"].numpy()) < 1e-10


def forecast_reference(mod, post_mean_last, post_cov_last, useq_future, H):
    """State forecasts x_k = A x_{k-1} + u[T + k - 1], S_k = A S_{k-1} A' + P from the last smoothed posterior
    (post_mean_last[d, batch], post_cov_last[d, d, batch]); useq_future = rows T.. of the sequence ([H, d] or
    [H, d, batch]).  Returns (mean[H, d, batch], cov[H, d, d, batch]) in fp64 numpy."""
    A, P = mod["A"].astype(np.float64), mod["P"].astype(np.float64)
    x = np.asarray(post_mean_last, np.float64); S = np.moveaxis(np.asarray(post_cov_last, np.float64), -1, 0)
    uf = np.asarray(useq_future, np.float64)
    uf = uf[..., None] if uf.ndim == 2 else uf
    ms, Ss = [], []
    for k in range(H):
        x = A @ x + uf[k]
        S = A @ S @ A.T + P
        ms.append(x); Ss.append(np.moveaxis(S, 0, -1))
    return np.stack(ms), np.stack(Ss)


@pytest.mark.parametrize("d,m", CASES)
@pytest.mark.parametrize("per_chain", [False, True])
def test_forecasts_are_the_smoother_on_padded_data(d, m, per_chain):
    """Forecast k = 1..H steps with row T + k - 1 of the inputs: the same as smoothing y padded with H missing steps and
    the same T + H input rows (1e-10)."""
    mod = random_model(d, m, seed=60 + 10 * d + m)
    T, H, nb = 14, 4, 5
    y = simulate(mod, T, nb, seed=d + 9 * m)
    useq = input_sequence(T + H, d, seed=11, nb=nb if per_chain else None)
    yp = np.concatenate([y, np.zeros((H, m, nb), np.float32)])
    mask = np.ones((T + H, nb), np.uint8); mask[T:] = 0
    pad = kalman_rts_inputs(per_chain_models(mod, nb), torch.as_tensor(yp), useq, mask=mask)
    sm = kalman_rts_inputs(per_chain_models(mod, nb), torch.as_tensor(y), useq[:T])
    fm, fc = forecast_reference(mod, sm["mean"][-1].numpy(), sm["cov"][-1].numpy(), useq[T:], H)
    assert _rel(sm["mean"].numpy(), pad["mean"][:T].numpy()) < 1e-10
    assert _rel(fm, pad["mean"][T:].numpy()) < 1e-10
    assert _rel(fc, pad["cov"][T:].numpy()) < 1e-10


def test_reference_without_inputs_is_the_variant_reference():
    """With a zero sequence the gain-table form is the reference of test_shared_sweep_variants bit for bit."""
    mod = random_model(4, 4, seed=5)
    y = torch.as_tensor(simulate(mod, 30, 7, seed=1))
    a = input_reference(mod, y, np.zeros((30, 4)), transition_first=True)
    b = reference_sweep(mod, y, transition_first=True)
    assert torch.equal(a["mean"], b["mean"]) and torch.equal(a["nle"], b["nle"])


# ====================================================================================== CPU: argument handling
def _bare_context():
    from rxinfer_jl_b200.context import Context
    return object.__new__(Context)         # no device: only the host-side argument handling runs


def test_context_inputs_argument_rules(rx):
    from rxinfer_jl_b200 import _lib as L
    c = _bare_context()
    T, d, nb = 6, 3, 4
    assert c._inputs(None, None, T, d, nb) is None
    flag, ptr, keep = c._inputs(np.ones((T, d)), None, T, d, nb)
    assert flag == L.U_SEQ_SHARED and keep.dtype == np.float32 and keep.flags.c_contiguous
    flag, _, _ = c._inputs(torch.ones(T, d), None, T, d, nb)               # a CPU tensor is a host sequence
    assert flag == L.U_SEQ_SHARED
    with pytest.raises(ValueError, match="either a constant offset"):
        c._inputs(np.ones((T, d)), np.ones(d), T, d, nb)
    with pytest.raises(ValueError, match="expected a host array of shape"):
        c._inputs(np.ones((T - 1, d)), None, T, d, nb)                      # predict needs T + H rows: rows is checked
    with pytest.raises(ValueError, match="expected a host array of shape"):
        c._inputs(np.ones((T, d, nb)), None, T, d, nb)                      # a per-chain sequence must be a CUDA tensor
    assert L.U_SEQ_SHARED == 1 << 8 and L.U_SEQ_CHAIN == 1 << 9


def test_header_declares_the_input_flags():
    import os
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    h = open(os.path.join(root, "include", "rxgauss.h")).read()
    assert "RXG_U_SEQ_SHARED    = 1u << 8" in h and "RXG_U_SEQ_CHAIN     = 1u << 9" in h


def _lgssm_model(rx, smoothing=True, **kw):
    from rxinfer_jl_b200 import inference as I
    mod = random_model(2, 2, seed=1)
    cls = I.linear_gaussian_ssm_smoothing if smoothing else I.linear_gaussian_ssm_filtering
    return cls(A=mod["A"], B=mod["B"], P=mod["P"], Q=mod["Q"], x0=(mod["m0"], mod["S0"]), **kw)


def test_infer_inputs_argument_rules(rx):
    """data['u'] with a constant model.u, a wrong row count with a horizon, and inputs on a model without a transition
    input are refused before any device work."""
    from rxinfer_jl_b200 import inference as I
    y = torch.zeros(5, 2, 3)
    with pytest.raises(ValueError, match="fold the constant"):
        I.infer(model=_lgssm_model(rx, u=np.ones(2)), data={"y": y, "u": np.zeros((5, 2))})
    with pytest.raises(ValueError, match="fold the constant"):
        I.infer(model=_lgssm_model(rx, smoothing=False, u=np.ones(2)), data={"y": y, "u": np.zeros((5, 2))})
    with pytest.raises(ValueError, match="T \\+ horizon"):
        I.infer(model=_lgssm_model(rx, horizon=2), data={"y": y, "u": np.zeros((5, 2))})
    with pytest.raises(NotImplementedError, match="belong to the LGSSM"):
        I.infer(model=I.hgf(), data={"y": torch.zeros(5, 3), "u": np.zeros((5, 1))})


def test_predictvars_with_inputs(rx):
    """A bare KeepLast() predicts the observations, not the known inputs; asking for 'u' explicitly is refused."""
    from rxinfer_jl_b200 import inference as I
    model = _lgssm_model(rx)
    data = {"y": torch.zeros(5, 2, 3), "u": np.zeros((5, 2))}
    assert I._predict_keys(I.KeepLast(), model, data) == {"y"}
    with pytest.raises(NotImplementedError, match="known inputs"):
        I._predict_keys({"u": I.KeepLast()}, model, data)


# ====================================================================================== Julia shim (structure only)
def _shim():
    import os
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    return open(os.path.join(root, "rxinfer.jl_b200", "julia", "RxGaussB200.jl")).read()


def test_julia_shim_binds_the_input_flags():
    s = _shim()
    assert "const RXG_U_SEQ_SHARED     = UInt32(1) << 8" in s
    assert "const RXG_U_SEQ_CHAIN      = UInt32(1) << 9" in s


def test_julia_recognise_handles_data_inputs():
    """`recognise` conditions the graph on `u` as well, accepts a `+` node whose operand is a data variable and reports
    it in the pattern (`u_data`); `infer_batched` packs the shared or per-series form and passes it to the sweep."""
    s = _shim()
    body = s[s.index("function recognise(generator, one_series; inputs = nothing)"):s.index("\"\"\"\n    infer_batched")]
    assert "(y = one_series, u = inputs)" in body
    assert "data_operand(model, props)" in body and "ndata > 0" in body
    assert "u_data::Bool" in s
    ib = s[s.index("function infer_batched"):]
    ib = ib[:ib.index("\nend\n")]
    assert "RXG_U_SEQ_CHAIN" in s and "sweep_chain_inputs" in s
    assert "inputs = us === nothing ? nothing : first(us)" in ib
    assert "sweep(context, pattern, y; mask, free_energy = free_energy !== false, inputs)" in ib


def test_julia_stock_forwards_every_data_key():
    """The fallback runs stock RxInfer with every data key of the series (y, u, ...), not only y."""
    s = _shim()
    ib = s[s.index("function infer_batched"):]
    ib = ib[:ib.index("\nend\n")]
    assert "data = (y = ys[b],)" not in ib
    assert "series(b) = NamedTuple{keys(data)}(map(v -> v[b], values(data)))" in ib
    assert "data = series(b)" in ib
