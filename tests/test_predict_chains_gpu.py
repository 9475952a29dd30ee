"""The prediction post-pass of rxg_lgssm_smooth_predict_f32 (csrc/rxg_predict.cu, DESIGN section 3.12) step by step and
chain by chain, against fp64, on both routes and across their launch edges.

Two references, both fp64 torch batched over chains (`post_pass`):
  (a) the closed form evaluated on the device's OWN outputs of the same call (posterior means and covariances, state
      forecasts) and the fp32-rounded model: it isolates the post-pass, so smoother error cannot hide an error in it.
      Route A (shared model) reads the chain-independent covariance table, route B every chain's own covariance.
  (b) the same closed form on the fp64 Kalman + RTS posteriors of the fp32-rounded model (end to end).
Every (step, chain, element) is gated against (a):
  * fp32 arithmetic (route A means: k_predict_mean_small or the MODE 1 / MODE 2 left-GEMM): |err| <= C u32 (|F||y| +
    |G||mu|) with F = I - K, G = K B from (a);
  * the forecast means (k_forecast_mean): |err| <= C beta_k, beta_k = |A| beta_{k-1} + gamma_d (|A||x_{k-1}| + |u_k|);
  * fp64 arithmetic stored in fp32 (k_predict_msg on both routes, k_forecast_cov): |err| <= C (u32 |ref| + u64 g ||.||),
    g = kappa(D_t) = (||Q|| + ||B S B'||) ||D_t^-1|| at an observed step (D_t = Q - B S B' is formed from nearly equal
    operands), d at a missing step, (k + 1) d for forecast k.
and every chain against (b) by relative L2 over steps at TOL_MEAN / TOL_COV (the conditioning-stress model and a
one-step series keep their own mean gates: the fp32 posterior error amplified by K_t, which (a) shows is not the
post-pass's).  The worst case of every (output, route,
shape) is printed at the end.  The CPU half checks reference (a) against both oracles and pins a Python restatement of
the launch geometry, so that the GPU cases provably land on its edges.
"""
import numpy as np
import pytest
import torch

from oracle.predict import predict_closed_form, predict_reference_schedule
from test_inputs import input_sequence, kalman_rts_inputs, per_chain_models
from test_shared_sweep_variants import NATIVE, per_chain_rel, random_model, simulate
from util import TOL_COV, TOL_MEAN, f32_model

U32, U64 = 2.0 ** -24, 2.0 ** -53
F64 = torch.float64
KEYS = ("A", "B", "P", "Q", "m0", "S0")
STRESS_TOL_MEAN = 1e-3        # end-to-end mean gate of the conditioning-stress model (DESIGN section 5)
# end-to-end mean gate of a one-step series (T = 1): a chain's m predictions carry the fp32 posterior error through
# K_t = Q D_t^-1 without any other step to pool it with (measured 2.1e-5 at d = m = 4, DESIGN section 5)
ONE_STEP_TOL_MEAN = 1e-4

# Gate constants: about 4x the worst ratio measured on one H100 80GB HBM3 at 700 W (DESIGN section 5): 4.43 (route A
# means, at 40 x 33), 0.98 (forecast means, d = 1), 0.999 (fp64 results stored in fp32: their rounding).
C_MEAN32 = 18.0               # route A means, error / (u32 (|F||y| + |G||mu|))
C_FC_MEAN = 4.0               # forecast means, error / beta_k
C_F64 = 4.0                   # k_predict_msg and k_forecast_cov outputs, error / (u32 |ref| + u64 g ||.||)

# ====================================================================================== launch geometry (rxg_predict.cu)
PW_MAX_WARPS, PM_TC, FM_THREADS, GRID_Y = 8, 16, 64, 65535    # warps, steps per CTA, chains per CTA, grid-y cap


def msg_layout_bytes(d, m):
    """Per-warp shared memory of k_predict_msg (msg_layout): fp64 R1, D, v; fp32 S_s, B, Q; 16-byte multiple."""
    r1 = max(m * (d + 1), m * (m + 1))
    nd = r1 + m * (m + 1) + 2 * m
    nf = d * (d + 1) + m * (d + 1) + m * (m + 1)
    return (nd * 8 + nf * 4 + 15) // 16 * 16


def msg_warps(d, m):
    """Warps (= items) per CTA of k_predict_msg."""
    return min(PW_MAX_WARPS, max(1, 49152 // msg_layout_bytes(d, m)))


def forecast_cov_opt_in(d):
    """k_forecast_cov needs the shared-memory opt-in above the 48 KiB default."""
    return 24 * d * (d + 1) > 48 * 1024


def left_gemm_mmax(M):
    return 16 if M <= 16 else (32 if M <= 32 else 64)


def route_b_batch(d, m, L, delta, base=9):
    """The smallest batch >= base whose L * batch k_predict_msg items sit at k nw + delta (L coprime to nw)."""
    nw = msg_warps(d, m)
    b = base
    while (L * b - delta) % nw:
        b += 1
    return b


# ====================================================================================== reference (a) / (b)
def _t(a, dev):
    return (a if isinstance(a, torch.Tensor) else torch.as_tensor(np.asarray(a, np.float64))).to(dev, F64)


def _mats(a, dev):
    """A shared matrix [r, c] or per-chain matrices [nb, r, c] -> [1 | nb, r, c]."""
    a = _t(a, dev)
    return a[None] if a.dim() == 2 else a


def _sym(S):
    return 0.5 * (S + S.transpose(-1, -2))


def _bmv(M, x):
    return (M @ x[..., None])[..., 0]


def post_pass(mod, y, obs, mean, cov, H=0, u=None, useq=None, fc_mean=None, fc_cov=None):
    """The closed form of DESIGN section 3.12 in fp64, batched over chains, in the ABI layouts (chain index last).

    mod: A, B, P, Q shared ([r, c]) or per chain ([nb, r, c]); y[T, m, nb]; obs[T, nb] (bool); mean[T, d, nb] and
    cov[T, d, d, nc] (nc = 1: the chain-independent table of route A; nc = nb: every chain's own) -- the posteriors the
    predictions are computed from.  u: constant offset [d] or per chain [nb, d]; useq: input rows [T + H, d] or
    [T + H, d, nb] (forecast k uses row T + k - 1).  fc_mean[H, d, nb] / fc_cov[H, d, d, nc]: state forecasts the
    forecast-row predictions are computed from (the device's own; default: this recursion's).

    Returns pred_mean[T+H, m, nb], pred_cov[T+H, m, m, nc], fc_mean[H, d, nb], fc_cov[H, d, d, nc] and the bound
    ingredients: mean_scale = |F||y| + |G||mu| [T+H, m, nb], g_mean[T+H, nb], g_cov[T+H, nc], beta[H, d, nb], g_fc[H]."""
    dev = y.device
    T, m, nb = y.shape
    A, B, P, Q = (_mats(mod[k], dev) for k in "ABPQ")
    d = A.shape[-1]
    Y = y.to(dev, F64).permute(0, 2, 1)                                         # [T, nb, m]
    MU = _t(mean, dev).permute(0, 2, 1)                                          # [T, nb, d]
    S = _t(cov, dev)
    S = (S[..., None] if S.dim() == 3 else S).permute(0, 3, 1, 2)                # [T, nc, d, d]
    nc = S.shape[1]
    ob = torch.as_tensor(obs, device=dev).bool()
    if nc == 1:
        assert bool((ob == ob[:, :1]).all()), "a chain-independent table needs one missing-data pattern for every chain"
        ob = ob[:, :1]
    om = ob[..., None, None]
    Bt, At = B.transpose(-1, -2), A.transpose(-1, -2)
    BSB = _sym(B @ S @ Bt)
    D = Q - BSB
    X = torch.linalg.solve_ex(D, Q.expand(D.shape).contiguous())[0]               # D^-1 Q, K = Q D^-1 = X'
    K = X.transpose(-1, -2)
    eye = torch.eye(m, dtype=F64, device=dev)
    F = torch.where(om, eye - K, torch.zeros_like(K))
    G = torch.where(om, K @ B, B.expand(K.shape[:-2] + B.shape[-2:]))
    C = torch.where(om, _sym(Q @ X), BSB + Q)
    lmin = torch.cat([torch.linalg.eigvalsh(_sym(Dc))[..., 0] for Dc in D.split(4096)])
    kap = (torch.linalg.matrix_norm(Q, ord=2) + torch.linalg.matrix_norm(BSB, ord=2)) / lmin
    kap = torch.where(lmin > 0, kap, torch.full_like(kap, float("inf")))
    g_cov = torch.where(ob, kap, torch.full_like(kap, float(d)))                 # [T, nc]
    pm = _bmv(F, Y) + _bmv(G, MU)                                                # [T, nb, m]
    scale = _bmv(F.abs(), Y.abs()) + _bmv(G.abs(), MU.abs())

    # forecasts from (mu_s[T-1], S_s[T-1])
    uc = None
    if useq is not None:
        us = _t(useq, dev)
        us = (us[:, None, :] if us.dim() == 2 else us.permute(0, 2, 1))          # [T+H, 1 | nb, d]
    elif u is not None:
        uc = _t(u, dev)
        uc = uc[None] if uc.dim() == 1 else uc                                   # [1 | nb, d]
    x, Sx = MU[T - 1], S[T - 1]
    beta = torch.zeros_like(x)
    gd = d * U32 / (1.0 - d * U32)
    fm, fS, fb = [], [], []
    for k in range(H):
        uk = us[T + k] if useq is not None else (uc if uc is not None else torch.zeros(1, d, dtype=F64, device=dev))
        beta = _bmv(A.abs(), beta) + gd * (_bmv(A.abs(), x.abs()) + uk.abs())
        x = _bmv(A, x) + uk
        Sx = _sym(A @ Sx @ At + P)
        fm.append(x); fS.append(Sx); fb.append(beta)
    out = dict(F=F, G=G)
    if H:
        fm, fS, fb = torch.stack(fm), torch.stack(fS), torch.stack(fb)           # [H, nb, d], [H, nc, d, d]
        xin = fm if fc_mean is None else _t(fc_mean, dev).permute(0, 2, 1)
        Sin = fS if fc_cov is None else _t(fc_cov, dev)
        if fc_cov is not None:
            Sin = (Sin[..., None] if Sin.dim() == 3 else Sin).permute(0, 3, 1, 2)
        pm = torch.cat([pm, _bmv(B, xin)])
        scale = torch.cat([scale, _bmv(B.abs(), xin.abs())])
        C = torch.cat([C, _sym(B @ Sin @ Bt) + Q])
        g_cov = torch.cat([g_cov, torch.full((H, g_cov.shape[1]), float(d), dtype=F64, device=dev)])
        out.update(fc_mean=fm.permute(0, 2, 1), fc_cov=fS.permute(0, 2, 3, 1), beta=fb.permute(0, 2, 1),
                   g_fc=(torch.arange(H, dtype=F64, device=dev) + 1.0) * d)
    out.update(pred_mean=pm.permute(0, 2, 1), pred_cov=C.permute(0, 2, 3, 1), mean_scale=scale.permute(0, 2, 1),
               g_cov=g_cov, g_mean=g_cov.expand(T + H, nb))
    return out


def oracle_posteriors(mod, y, obs, useq, per_chain, tf):
    """fp64 Kalman + RTS posteriors (mean[T, d, nb], cov[T, d, d, nb]) of the fp32-rounded model on y's device."""
    T, m, nb = y.shape
    dev = y.device
    mods = ({k: _t(mod[k], dev) for k in KEYS} if per_chain else per_chain_models(mod, nb, dev))
    return kalman_rts_inputs(mods, y, useq, mask=obs, transition_first=tf)


def end_to_end(mod, y, obs, H, u, useq, per_chain, tf):
    """Reference (b): the closed form on the oracle's posteriors."""
    T, m, nb = y.shape
    d = np.asarray(mod["A"]).shape[-1]
    rows = useq
    if rows is None:
        if u is None:
            rows = np.zeros((T + H, d))
        else:
            uu = np.asarray(u, np.float64)
            rows = np.repeat(uu[None], T + H, 0) if uu.ndim == 1 else torch.as_tensor(np.repeat(uu.T[None], T + H, 0))
    post_rows = rows[:T]
    ora = oracle_posteriors(mod, y, obs, post_rows, per_chain, tf)
    out = post_pass(mod, y, obs, ora["mean"], ora["cov"], H, useq=rows)
    out["mean"] = ora["mean"]
    return out


# ====================================================================================== CPU: the references
def _rel(a, b):
    a = np.asarray(a, np.float64); b = np.asarray(b, np.float64)
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-300))


def _cpu_model(rng, d, m):
    A = 0.9 * np.linalg.qr(rng.standard_normal((d, d)))[0]
    B = rng.standard_normal((m, d))
    G = rng.standard_normal((d, d)); P = G @ G.T / d + 0.1 * np.eye(d)
    G = rng.standard_normal((m, m)); Q = G @ G.T / m + 0.5 * np.eye(m)
    return dict(A=A, B=B, P=P, Q=Q, m0=rng.standard_normal(d), S0=2.0 * np.eye(d))


def _cpu_mask(T, nb, rng):
    mask = rng.random((T, nb)) > 0.3
    mask[-3:, 0] = False
    mask[:, 1] = False
    mask[:, 2] = True
    return mask


@pytest.mark.parametrize("d,m", [(1, 1), (4, 4), (4, 3), (3, 5), (6, 2)])
@pytest.mark.parametrize("H", [0, 3])
@pytest.mark.parametrize("with_u", [False, True])
def test_reference_matches_the_closed_form_oracle(d, m, H, with_u):
    """Reference (a) fed the oracle's fp64 posteriors = oracle/predict.py::predict_closed_form (1e-12)."""
    rng = np.random.default_rng(7 * d + m + 100 * H)
    mod = _cpu_model(rng, d, m)
    T, nb = 13, 6
    u = rng.standard_normal(d) if with_u else None
    y = rng.standard_normal((T, m, nb))
    mask = _cpu_mask(T, nb, rng)
    c = predict_closed_form(y, **mod, mask=mask, u=u, horizon=H)
    r = post_pass(mod, torch.as_tensor(y), torch.as_tensor(mask), c["mean"], c["cov"], H, u=u)
    for k in ("pred_mean", "pred_cov") + (("fc_mean", "fc_cov") if H else ()):
        assert _rel(r[k].numpy(), c[k]) < 1e-12, k


@pytest.mark.parametrize("d,m", [(1, 1), (4, 4), (4, 3), (3, 5)])
@pytest.mark.parametrize("H", [0, 3])
def test_reference_matches_the_schedule_oracle(d, m, H):
    """Reference (a) on the rule-built oracle's posteriors = predict_reference_schedule (1e-10), at the shapes
    tests/test_predict.py uses, and the chain-independent table form (nc = 1) = the per-chain form."""
    rng = np.random.default_rng(100 * d + 10 * m + H)
    mod = _cpu_model(rng, d, m)
    u = rng.standard_normal(d)
    T, nb = 11, 6
    y = rng.standard_normal((T, m, nb))
    mask = _cpu_mask(T, nb, rng)
    s = predict_reference_schedule(y, **mod, mask=mask, u=u, horizon=H)
    r = post_pass(mod, torch.as_tensor(y), torch.as_tensor(mask), s["mean"], s["cov"], H, u=u)
    for k in ("pred_mean", "pred_cov") + (("fc_mean", "fc_cov") if H else ()):
        assert _rel(r[k].numpy(), s[k]) < 1e-10, k
    tm = np.ones(T, bool); tm[0] = tm[5] = tm[-1] = False
    full = np.repeat(tm[:, None], nb, 1)
    s = predict_reference_schedule(y, **mod, mask=full, u=u, horizon=H)
    r = post_pass(mod, torch.as_tensor(y), torch.as_tensor(full), s["mean"], s["cov"][..., :1], H, u=u)
    assert _rel(r["pred_mean"].numpy(), s["pred_mean"]) < 1e-10
    assert _rel(np.broadcast_to(r["pred_cov"].numpy(), s["pred_cov"].shape), s["pred_cov"]) < 1e-10


@pytest.mark.parametrize("per_chain_seq", [False, True])
def test_end_to_end_reference_with_inputs(per_chain_seq):
    """Reference (b) with an input sequence = the smoother on y padded with H missing steps and the same T + H rows."""
    mod = f32_model(random_model(3, 2, 5))
    T, H, nb = 12, 4, 5
    y = torch.as_tensor(simulate(mod, T, nb, 6))
    useq = input_sequence(T + H, 3, 8, nb if per_chain_seq else None)
    obs = torch.ones(T, nb, dtype=torch.bool); obs[4, 2] = False
    r = end_to_end(mod, y, obs, H, None, useq, False, False)
    yp = torch.cat([y, torch.zeros(H, 2, nb, dtype=y.dtype)])
    op = torch.cat([obs, torch.zeros(H, nb, dtype=torch.bool)])
    pad = kalman_rts_inputs(per_chain_models(mod, nb), yp, useq, mask=op)
    assert _rel(r["fc_mean"].numpy(), pad["mean"][T:].numpy()) < 1e-10
    assert _rel(r["fc_cov"].numpy(), pad["cov"][T:].numpy()) < 1e-10
    B, Q = mod["B"], mod["Q"]
    pm = np.einsum("kd,tdb->tkb", B, pad["mean"][T:].numpy())
    assert _rel(r["pred_mean"][T:].numpy(), pm) < 1e-10
    pc = np.einsum("kd,tdeb,le->tklb", B, pad["cov"][T:].numpy(), B) + Q[None, :, :, None]
    assert _rel(r["pred_cov"][T:].numpy(), pc) < 1e-10


def test_launch_geometry_restatement():
    """The restated formulas of rxg_predict.cu / rxg_rules_large.cu put the GPU cases below on the launch edges."""
    assert [msg_warps(k, k) for k in (1, 4, 6, 16, 20, 24, 31, 32, 33, 40, 64)] == [8, 8, 8, 6, 4, 2, 1, 1, 1, 1, 1]
    assert msg_layout_bytes(64, 64) == 117504                                 # "117 KB, one warp" (DESIGN 3.12)
    assert msg_layout_bytes(4, 4) == 624 and msg_layout_bytes(16, 16) == 7872
    assert [forecast_cov_opt_in(d) for d in (1, 44, 45, 64)] == [False, False, True, True]
    assert [left_gemm_mmax(M) for M in (1, 16, 17, 32, 33, 64)] == [16, 16, 32, 32, 64, 64]
    assert PM_TC * GRID_Y == 1048560                                          # rows before the grid-y loop's second lap
    for d, m in ROUTE_B_SHAPES:
        nw = msg_warps(d, m)
        for delta in (-1, 0, 1):
            b = route_b_batch(d, m, 13, delta)
            assert (13 * b - delta) % nw == 0 and b >= 9


# ====================================================================================== GPU: running and gating
WORST = {}      # (output, route, shape) -> (ratio or error, where)


def _record(key, value, where):
    if key not in WORST or value > WORST[key][0]:
        WORST[key] = (float(value), where)


@pytest.fixture(scope="module", autouse=True)
def _report_worst(request):
    yield
    if not WORST:
        return
    with request.config.pluginmanager.getplugin("capturemanager").global_and_fixture_disabled():
        print("\nprediction post-pass, worst case per (output, route, shape) (post-pass gates: error / bound; "
              "end to end: per-chain relative L2):")
        for key in sorted(WORST):
            v, where = WORST[key]
            print(f"  {key[0]:<16s} {key[1]:<2s} {key[2]:<8s} {v:.3e}  ({where})")


def gate(name, route, shp, case, got, ref, bound, limit, t0=0):
    """|got - ref| <= limit * bound for every element; got / ref / bound in the ABI layout (row first, chain last); t0 is
    the step of row 0."""
    got = got.to(ref.device, F64)
    err = (got - ref).abs()
    ratio = torch.where(err == 0, torch.zeros_like(err), err / bound)
    ratio = torch.nan_to_num(ratio, nan=float("inf"))
    flat = int(ratio.argmax())
    v = float(ratio.flatten()[flat])
    idx = tuple(int(i) for i in np.unravel_index(flat, tuple(ratio.shape)))
    where = f"{name} t = {idx[0] + t0}, chain {idx[-1]}, {idx[1:-1]}"
    _record((name, route, shp), v, f"{case}: {where}")
    assert v <= limit, (f"{case}: {where}: |{float(got[idx]):.9g} - {float(ref[idx]):.9g}| = {float(err[idx]):.3e} is "
                        f"{v:.3e} x its bound (limit {limit:g})")


def _rowmax(x, nd):
    """max |x| over the element axes (1 .. nd) of an ABI-layout tensor, kept broadcastable."""
    r = x.abs()
    for ax in range(1, nd + 1):
        r = r.amax(ax, keepdim=True)
    return r


def gate_post_pass(route, shp, case, r, a, H, T):
    """Every output of one call against reference (a)."""
    nb = r["pred_mean"].shape[-1]
    pm = a["pred_mean"]
    g_mean = a["g_mean"][:, None, :]
    if route == "A":
        # chain-independent table (F_t, G_t) applied in fp32: observed, missing and forecast rows alike
        gate("pred_mean", route, shp, case, r["pred_mean"], pm, U32 * a["mean_scale"], C_MEAN32)
    else:
        sc = _rowmax(a["mean_scale"], 1)
        gate("pred_mean", route, shp, case, r["pred_mean"], pm, U32 * pm.abs() + U64 * g_mean * sc, C_F64)
    pc = r["pred_cov"]
    if pc is not None:
        if pc.dim() == 3:
            pc = pc[..., None]
        if route == "A":
            pc = pc[..., :1]
        rc = a["pred_cov"]
        gate("pred_cov", route, shp, case, pc, rc, U32 * rc.abs() + U64 * a["g_cov"][:, None, None, :] * _rowmax(rc, 2),
             C_F64)
    if H and r["fc_mean"] is not None:
        gate("fc_mean", route, shp, case, r["fc_mean"], a["fc_mean"], a["beta"], C_FC_MEAN)
        fc = r["fc_cov"]
        fc = fc[..., None] if fc.dim() == 3 else fc
        if route == "A":
            fc = fc[..., :1]
        rf = a["fc_cov"]
        gate("fc_cov", route, shp, case, fc, rf, U32 * rf.abs() + U64 * a["g_fc"][:, None, None, None] * _rowmax(rf, 2),
             C_F64)


def gate_end_to_end(route, shp, case, r, b, H, tol_mean=TOL_MEAN):
    """Every chain against reference (b), relative L2 over steps.  The forecast states are gated together with the
    chain's posterior means (one state trajectory of T + H steps): a forecast of a state near 0 has no relative scale."""
    pairs = [("pred_mean", r["pred_mean"], b["pred_mean"], tol_mean), ("pred_cov", r["pred_cov"], b["pred_cov"], TOL_COV)]
    if H and r["fc_mean"] is not None:
        pairs += [("fc_mean", torch.cat([r["mean"], r["fc_mean"]]), torch.cat([b["mean"].to(F64), b["fc_mean"]]), TOL_MEAN),
                  ("fc_cov", r["fc_cov"], b["fc_cov"], TOL_COV)]
    for k, got, ref, tol in pairs:
        if got is None:
            continue
        if got.dim() == ref.dim() - 1:
            got = got[..., None]
        err = per_chain_rel(got.expand(ref.shape) if got.shape[-1] == 1 else got, ref)
        c = int(err.argmax()); e = float(err[c])
        _record((k + " e2e", route, shp), e, f"{case}: chain {c}")
        assert e < tol, f"{case}: {k} relative L2 of chain {c} against the end-to-end reference = {e:.3e} >= {tol:g}"


def _dev_model(mod):
    return {k: torch.as_tensor(np.ascontiguousarray(np.moveaxis(np.asarray(v, np.float32), 0, -1)), device="cuda")
            for k, v in mod.items()}


def run(ctx, mod, y, *, H, mask=None, u=None, useq=None, per_chain=False, **kw):
    """One rxg_lgssm_smooth_predict_f32 call.  mod: fp32-rounded fp64 numpy, shared or per chain ([nb, ...]); mask: a
    shared [T] numpy pattern or a [T, nb] uint8 CUDA tensor; u: [d] or per chain [nb, d]; useq: host [T + H, d] or CUDA
    [T + H, d, nb]."""
    if per_chain:
        D = _dev_model({k: mod[k] for k in KEYS})
        args = [D[k] for k in KEYS]
        ud = None if u is None else torch.as_tensor(np.ascontiguousarray(np.asarray(u, np.float32).T), device="cuda")
    else:
        args = [mod[k] for k in KEYS]
        ud = u
    r = ctx.lgssm_predict(y, *args, horizon=H, u=ud, inputs=useq, mask=mask, per_chain_model=per_chain,
                          want_status=True, **kw)
    torch.cuda.synchronize()
    return r


def _obs(mask, T, nb):
    if mask is None:
        return torch.ones(T, nb, dtype=torch.bool, device="cuda")
    if isinstance(mask, np.ndarray):
        return torch.as_tensor(mask.astype(bool), device="cuda")[:, None].expand(T, nb)
    return mask.bool()


def check(ctx, route, mod, y, *, H, mask=None, u=None, useq=None, per_chain=False, tf=False, e2e=True,
          tol_mean=TOL_MEAN, case="", **kw):
    """Run one call and gate it against (a) and, with e2e, (b).  Returns the call's outputs."""
    T, m, nb = y.shape
    d = np.asarray(mod["A"]).shape[-1]
    shp = f"{d}x{m}"
    r = run(ctx, mod, y, H=H, mask=mask, u=u, useq=useq, per_chain=per_chain, transition_first=tf, **kw)
    st = r["status"]
    assert int((st != 0).sum()) == 0, f"{case}: chains flagged {torch.nonzero(st).flatten().tolist()[:8]}"
    obs = _obs(mask, T, nb)
    cov, fc_cov = r["cov"], r["fc_cov"]
    if route == "A":                                                # route A reads chain 0 / the table
        cov = cov[..., :1] if cov.dim() == 4 else cov
        fc_cov = fc_cov[..., :1] if fc_cov is not None and fc_cov.dim() == 4 else fc_cov
    a = post_pass(mod, y, obs, r["mean"], cov, H, u=u, useq=useq, fc_mean=r["fc_mean"], fc_cov=fc_cov)
    gate_post_pass(route, shp, case, r, a, H, T)
    if e2e:
        b = end_to_end(mod, y, obs, H, u, useq, per_chain, tf)
        gate_end_to_end(route, shp, case, r, b, H, tol_mean)
    return r


def _pattern(T):
    """Shared missing-data pattern: first and last step missing; from T = 20 a gap across the first 16-step tile edge,
    from T = 40 a missing step right after the second (the observed step 31 is the last of its tile)."""
    tm = np.ones(T, np.uint8)
    tm[0] = 0
    tm[-1] = 0
    if T >= 20:
        tm[14:18] = 0
    if T >= 40:
        tm[32] = 0
    return tm


def _y(mod, T, nb, seed):
    return torch.as_tensor(simulate(mod, T, nb, seed), device="cuda")


def _equal_outputs(r1, r2, keys=("mean", "cov", "pred_mean", "pred_cov", "fc_mean", "fc_cov"), sel=None):
    for k in keys:
        a, b = r1[k], r2[k]
        if a is None and b is None:
            continue
        if sel is not None:
            a, b = a[..., sel], b[..., sel]
        assert torch.equal(a, b), k


# ---------------------------------------------------------------------------------------------- route A, register means
REG_COMBOS = [(1, 0, 63), (15, 1, 64), (16, 17, 65), (17, 0, 255), (40, 17, 256), (40, 1, 257), (17, 100, 64)]


@pytest.mark.gpu
@pytest.mark.parametrize("masked", [False, True])
@pytest.mark.parametrize("d,m", NATIVE)
def test_register_means(ctx, d, m, masked):
    """k_predict_mean_small at every native shape: T = 1, 15, 16, 17, 40 puts t = T inside and on a 16-step tile;
    batches 63 ... 257 cross the 64-chain forecast CTA and the 256-chain mean CTA; H = 0, 1, 17, 100."""
    mod = f32_model(random_model(d, m, 10 * d + m))
    for i, (T, H, nb) in enumerate(REG_COMBOS):
        u = (0.3 * np.arange(1, d + 1) / d).astype(np.float32).astype(np.float64) if i % 2 else None
        tm = _pattern(T) if masked else None
        y = _y(mod, T, nb, i)
        r = check(ctx, "A", mod, y, H=H, mask=tm, u=u, tf=(i == 2), tol_mean=ONE_STEP_TOL_MEAN if T == 1 else TOL_MEAN,
                  case=f"T={T} H={H} batch={nb}")
        assert torch.equal(r["pred_cov"], r["pred_cov"][..., :1].expand_as(r["pred_cov"]))
        if H:
            assert torch.equal(r["fc_cov"], r["fc_cov"][..., :1].expand_as(r["fc_cov"]))
    # the same last call with the covariance table outputs, without prediction / forecast covariances, without post_cov
    tab = run(ctx, mod, y, H=H, mask=tm, u=u, cov_shared_out=True)
    assert torch.equal(r["pred_cov"], tab["pred_cov"][..., None].expand_as(r["pred_cov"]))
    assert torch.equal(r["fc_cov"], tab["fc_cov"][..., None].expand_as(r["fc_cov"]))
    lean = run(ctx, mod, y, H=H, mask=tm, u=u, want_pred_cov=False, want_forecast_states=False)
    nocov = run(ctx, mod, y, H=H, mask=tm, u=u, want_cov=False)
    for k in ("pred_mean", "fc_mean"):
        assert torch.equal(r[k], tab[k]), k
    assert torch.equal(r["pred_mean"], lean["pred_mean"])
    # without post_cov the family's own table feeds the post-pass: the same bits as chain 0 of post_cov
    _equal_outputs(r, nocov, keys=("mean", "pred_mean", "pred_cov", "fc_mean", "fc_cov"))


# ---------------------------------------------------------------------------------------------- route A, left-GEMM means
GEMM_SHAPES = [(3, 2), (4, 3), (5, 3), (8, 8), (16, 16), (17, 17), (20, 12), (33, 20), (33, 33), (40, 33), (64, 64)]
GEMM_COMBOS = [(12, 3, 255, False), (5, 0, 256, True), (17, 1, 257, False), (3, 2, 513, True)]


@pytest.mark.gpu
@pytest.mark.parametrize("d,m", GEMM_SHAPES)
def test_left_gemm_means(ctx, d, m):
    """MODE 1 (Y = G_t mu_t) and MODE 2 (Y += F_t y_t) left-GEMM at m on both sides of 16 | 17 and 32 | 33, batches on
    both sides of the 256-column tile, per-chain and [T][d][d] covariance outputs."""
    mod = f32_model(random_model(d, m, 7 * d + m))
    for i, (T, H, nb, masked) in enumerate(GEMM_COMBOS):
        tm = _pattern(T) if masked else None
        u = (0.2 * np.ones(d)).astype(np.float32).astype(np.float64) if i % 2 else None
        y = _y(mod, T, nb, 30 + i)
        shared = i == 2
        r = check(ctx, "A", mod, y, H=H, mask=tm, u=u, cov_shared_out=shared, case=f"T={T} H={H} batch={nb}"
                  + (" cov_shared_out" if shared else ""))
        if not shared:
            assert torch.equal(r["pred_cov"], r["pred_cov"][..., :1].expand_as(r["pred_cov"]))
            if H:
                assert torch.equal(r["fc_cov"], r["fc_cov"][..., :1].expand_as(r["fc_cov"]))
    lean = run(ctx, mod, y, H=H, mask=tm, u=u, want_pred_cov=False, want_forecast_states=False)
    assert torch.equal(r["pred_mean"], lean["pred_mean"])


# ---------------------------------------------------------------------------------------------- route B
ROUTE_B_SHAPES = NATIVE + [(5, 3), (16, 16), (20, 20), (24, 24), (31, 31), (32, 32), (33, 33), (40, 33), (64, 64)]


def _per_chain_model(d, m, nb, seed):
    ms = [random_model(d, m, seed + b) for b in range(nb)]
    return {k: np.stack([x[k] for x in ms]) for k in KEYS}


def _per_chain_mask(T, nb, seed):
    rng = np.random.default_rng(seed)
    mk = (rng.random((T, nb)) > 0.3).astype(np.uint8)
    mk[-min(3, T):, 0] = 0                       # trailing gap
    mk[:, 1] = 0                                 # prior-only chain
    return torch.as_tensor(mk, device="cuda")


@pytest.mark.gpu
@pytest.mark.parametrize("d,m", ROUTE_B_SHAPES)
def test_route_b(ctx, d, m):
    """k_predict_msg with one warp per (step, chain): (T + H) batch = 13 batch items at k nw - 1, k nw, k nw + 1 of this
    shape's warps per CTA; a per-chain model with a per-chain mask and offset, the forced path with a shared input
    sequence, and a per-chain mask with a per-chain input sequence."""
    L = 13
    # per-chain model, per-chain mask, per-chain constant offset, transition_first
    nb = route_b_batch(d, m, L, -1)
    T, H = 12, 1
    mod = f32_model(_per_chain_model(d, m, nb, 1000 * d + m))
    u = f32_model({"u": 0.3 * np.random.default_rng(d).standard_normal((nb, d))})["u"]
    y = torch.as_tensor((1.5 * np.random.default_rng(m).standard_normal((T, m, nb))).astype(np.float32), device="cuda")
    check(ctx, "B", mod, y, H=H, mask=_per_chain_mask(T, nb, d + m), u=u, per_chain=True, tf=True,
          case=f"per-chain model T={T} H={H} batch={nb}")
    # the forced per-chain path on a shared model, with a shared input sequence
    nb = route_b_batch(d, m, L, 0)
    T, H = 10, 3
    mod = f32_model(random_model(d, m, 3 * d + m))
    useq = input_sequence(T + H, d, d * m).astype(np.float32)
    check(ctx, "B", mod, _y(mod, T, nb, 2), H=H, useq=useq, force_per_chain_path=True,
          case=f"forced path, shared inputs T={T} H={H} batch={nb}")
    # a per-chain mask on a shared model, with a per-chain input sequence
    nb = route_b_batch(d, m, L, 1)
    T, H = 9, 4
    useq = torch.as_tensor(input_sequence(T + H, d, d + 5 * m, nb), device="cuda")
    check(ctx, "B", mod, _y(mod, T, nb, 3), H=H, useq=useq, mask=_per_chain_mask(T, nb, 7),
          case=f"per-chain mask, per-chain inputs T={T} H={H} batch={nb}")


# ---------------------------------------------------------------------------------------------- forecasts
@pytest.mark.gpu
@pytest.mark.parametrize("route", ["A", "B"])
@pytest.mark.parametrize("d", [44, 45])
def test_forecast_shared_memory_edge(ctx, d, route):
    """k_forecast_cov below (d = 44) and above (d = 45) its shared-memory opt-in, 100 forecast steps, 65 chains (two
    k_forecast_mean CTAs)."""
    m, T, H, nb = 3, 6, 100, 65
    mod = f32_model(random_model(d, m, d))
    u = (0.1 * np.ones(d)).astype(np.float32).astype(np.float64)
    check(ctx, route, mod, _y(mod, T, nb, d), H=H, u=u, force_per_chain_path=(route == "B"), case=f"H={H} batch={nb}")


# ---------------------------------------------------------------------------------------------- long cases
@pytest.mark.gpu
def test_left_gemm_slice_split(ctx):
    """left_gemm_per_slice launches at most 65 535 slices: T = 65 600 needs a second launch of 65 slices."""
    d, m, T, nb = 5, 3, 65600, 3
    mod = f32_model(random_model(d, m, 53))
    tm = _pattern(T)
    tm[65530:65540] = 0                       # missing steps on both sides of the split
    check(ctx, "A", mod, _y(mod, T, nb, 1), H=2, mask=tm, e2e=False, case=f"T={T} batch={nb}")


@pytest.mark.gpu
def test_register_means_second_grid_lap(ctx):
    """k_predict_mean_small's grid-y loop takes a second lap from row 16 * 65 535 = 1 048 560 on: T = 8,
    H = 1 048 600.  The tail rows, the head rows and the first forecast steps are gated against (a)."""
    d = m = 1
    T, H, nb = 8, 1048600, 3
    mod = f32_model(random_model(d, m, 11))
    y = _y(mod, T, nb, 4)
    r = run(ctx, mod, y, H=H, u=np.array([0.25]))
    assert int((r["status"] != 0).sum()) == 0
    tail = PM_TC * GRID_Y - 40
    # head: the observed rows and the first 200 forecasts, from the device's own posteriors
    K = 200
    a = post_pass(mod, y, _obs(None, T, nb), r["mean"], r["cov"][..., :1], K, u=np.array([0.25]),
                  fc_mean=r["fc_mean"][:K], fc_cov=r["fc_cov"][:K, ..., :1])
    sub = {k: (v[:T + K] if k.startswith("pred") else v[:K]) if v is not None else None for k, v in r.items()}
    gate_post_pass("A", "1x1 lap", f"T={T} H={H}, rows < {T + K}", sub, a, K, T)
    # tail: rows past the first lap are forecasts, F = 0, G = B, the prediction of the device's own forecast states
    B, Q = float(mod["B"][0, 0]), float(mod["Q"][0, 0])
    fm = r["fc_mean"][tail - T:].to(F64)
    fc = r["fc_cov"][tail - T:, ..., :1].to(F64)
    ref_m = B * fm
    gate("pred_mean", "A", "1x1 lap", f"T={T} H={H}, rows >= {tail}", r["pred_mean"][tail:], ref_m,
         U32 * ref_m.abs(), C_MEAN32, t0=tail)
    ref_c = B * fc * B + Q
    gate("pred_cov", "A", "1x1 lap", f"T={T} H={H}, rows >= {tail}", r["pred_cov"][tail:, ..., :1], ref_c,
         U32 * ref_c.abs() + U64 * ref_c.abs(), C_F64, t0=tail)


# ---------------------------------------------------------------------------------------------- conditioning stress
def _stress_model(q=1e-2, p=1e2, w2=np.pi / 35):
    """Observation-dominated model: two rotation blocks (angles pi / 15 and w2), Q = q I, P = p I."""
    A = np.zeros((4, 4))
    c1, s1, c2, s2 = np.cos(np.pi / 15), np.sin(np.pi / 15), np.cos(w2), np.sin(w2)
    A[:2, :2] = [[c1, -s1], [s1, c1]]; A[2:, 2:] = [[c2, -s2], [s2, c2]]
    return f32_model(dict(A=A, B=np.diag([1.3, 0.7, 1.3, 0.7]), P=p * np.eye(4), Q=q * np.eye(4), m0=np.zeros(4),
                          S0=100.0 * np.eye(4)))


@pytest.mark.gpu
def test_conditioning_stress_post_pass(ctx):
    """Q = 1e-2 I, P = 1e2 I: end to end the means keep their documented 1e-3 gate (fp32 posteriors amplified by
    K_t ~ 1e4), but on the posteriors it was given the post-pass meets the tight gates."""
    mod = _stress_model()
    T, H, nb = 200, 3, 64
    y = torch.as_tensor((10.0 * np.random.default_rng(77).standard_normal((T, 4, nb))).astype(np.float32), device="cuda")
    check(ctx, "A", mod, y, H=H, tol_mean=STRESS_TOL_MEAN, case="stress Q = 1e-2 I, P = 1e2 I")


# ---------------------------------------------------------------------------------------------- exact relations
@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["register", "gemm", "B"])
def test_chain_order_and_sub_batch(ctx, kind):
    """Reversing the chains, or re-running a sub-batch, reproduces every chain's outputs bit for bit."""
    d, m = {"register": (4, 4), "gemm": (20, 12), "B": (5, 3)}[kind]
    T, H, nb = 21, 5, 257 if kind != "B" else 140
    if kind == "B":
        mod = f32_model(_per_chain_model(d, m, nb, 77))
        y = torch.as_tensor((1.5 * np.random.default_rng(1).standard_normal((T, m, nb))).astype(np.float32), device="cuda")
        mask = _per_chain_mask(T, nb, 3)
    else:
        mod = f32_model(random_model(d, m, 78))
        y = _y(mod, T, nb, 2)
        mask = _pattern(T)
    pc = kind == "B"
    full = run(ctx, mod, y, H=H, mask=mask, per_chain=pc)
    rev = lambda t: t.flip(-1).contiguous()
    rmod = {k: v[::-1].copy() for k, v in mod.items()} if pc else mod
    back = run(ctx, rmod, rev(y), H=H, mask=rev(mask) if pc else mask, per_chain=pc)
    for k in ("pred_mean", "pred_cov", "fc_mean", "fc_cov"):
        assert torch.equal(rev(full[k]), back[k]), k
    lo, hi = 63, 130                              # crosses the 64- and 128-chain edges of k_forecast_mean's CTAs
    assert hi <= nb
    smod = {k: v[lo:hi].copy() for k, v in mod.items()} if pc else mod
    sub = run(ctx, smod, y[..., lo:hi].contiguous(), H=H, mask=mask[:, lo:hi].contiguous() if pc else mask, per_chain=pc)
    for k in ("pred_mean", "pred_cov", "fc_mean", "fc_cov"):
        assert torch.equal(full[k][..., lo:hi], sub[k]), k


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["register", "gemm", "B"])
def test_masked_observations_are_never_read(ctx, kind):
    """y at masked steps is ignored: finite garbage (+-1e30) there leaves every output bit-identical to zeros there."""
    d, m = {"register": (4, 4), "gemm": (5, 3), "B": (4, 4)}[kind]
    T, H, nb = 37, 2, 129
    mod = f32_model(random_model(d, m, 91))
    y = _y(mod, T, nb, 5)
    if kind == "B":
        mask = _per_chain_mask(T, nb, 9)
        miss = (mask == 0)[:, None, :].expand(T, m, nb)
    else:
        mask = _pattern(T)
        miss = torch.as_tensor(mask == 0, device="cuda")[:, None, None].expand(T, m, nb)
    sign = torch.where(torch.arange(T * m * nb, device="cuda").reshape(T, m, nb) % 2 == 0, 1.0, -1.0)
    y0 = torch.where(miss, torch.zeros_like(y), y).contiguous()
    yg = torch.where(miss, 1e30 * sign, y).contiguous()
    kw = dict(H=H, mask=mask, want_evidence=True, force_per_chain_path=(kind == "B"))
    r0, rg = run(ctx, mod, y0, **kw), run(ctx, mod, yg, **kw)
    _equal_outputs(r0, rg, keys=("mean", "cov", "neg_log_evidence", "pred_mean", "pred_cov", "fc_mean", "fc_cov",
                                 "status"))


# ---------------------------------------------------------------------------------------------- flags
@pytest.mark.gpu
def test_route_b_flags_only_the_chain_whose_d_is_not_spd(rx, ctx):
    """One chain with the conditioning-stress model (its D_t = Q - B S_s B' loses every digit in fp32) at the last
    chain of the first forecast CTA: only that chain gets RXG_ERR_NOT_SPD, every other chain is bit-identical to the call
    without it."""
    d = m = 4
    T, H, nb, bad = 60, 2, 65, FM_THREADS - 1
    good = _per_chain_model(d, m, nb, 400)
    mixed = {k: v.copy() for k, v in good.items()}
    for k, v in _stress_model().items():
        mixed[k][bad] = v
    good, mixed = f32_model(good), f32_model(mixed)
    y = torch.as_tensor((10.0 * np.random.default_rng(8).standard_normal((T, m, nb))).astype(np.float32), device="cuda")
    r_good = run(ctx, good, y, H=H, per_chain=True)
    r_bad = run(ctx, mixed, y, H=H, per_chain=True)
    sm = ctx.lgssm(y, *_dev_model({k: mixed[k] for k in KEYS}).values(), per_chain_model=True, want_status=True)
    torch.cuda.synchronize()
    assert int((sm["status"] != 0).sum()) == 0                       # the smoother itself flags nothing
    st = r_bad["status"].cpu().numpy()
    assert st[bad] == rx._lib.RXG_ERR_NOT_SPD
    assert (np.delete(st, bad) == 0).all()
    assert int((r_good["status"] != 0).sum()) == 0
    others = torch.arange(nb, device="cuda") != bad
    _equal_outputs(r_good, r_bad, sel=others)


@pytest.mark.gpu
def test_route_a_flags_every_chain(rx, ctx):
    """A shared model whose D_t is not SPD on the covariance table flags every chain (route A: the context flag).
    With Q = 1e-4 I and P = 1e4 I the fp32 table S_s rounds B S_s B' onto Q: D_t = Q - B S_s B', formed in fp64 from
    the table, has a negative eigenvalue although the smoother itself flags nothing.  The synchronous call returns
    RXG_ERR_NOT_SPD; asynchronously, status[b] = RXG_ERR_NOT_SPD for every chain and the next synchronisation reports
    the flag once."""
    mod = _stress_model(1e-4, 1e4, np.pi / 15)
    args = [mod[k] for k in KEYS]
    T, nb = 20, 70
    y = torch.as_tensor((10.0 * np.random.default_rng(2).standard_normal((T, 4, nb))).astype(np.float32), device="cuda")
    sm = ctx.lgssm(y, *args, want_status=True, cov_shared_out=True)
    torch.cuda.synchronize()
    assert int((sm["status"] != 0).sum()) == 0                       # the smoother itself flags nothing
    tab = sm["cov"].double().cpu().numpy()
    lmin = min(np.linalg.eigvalsh(mod["Q"] - mod["B"] @ tab[t] @ mod["B"].T)[0] for t in range(T))
    assert lmin <= 0.0, f"the model no longer gives a non-SPD D_t on the table (smallest eigenvalue {lmin:.3e})"
    with pytest.raises(rx.RxGaussError) as e:
        ctx.lgssm_predict(y, *args, horizon=1, want_status=True)
    assert e.value.code == rx._lib.RXG_ERR_NOT_SPD
    r = ctx.lgssm_predict(y, *args, horizon=1, want_status=True, asynchronous=True)
    with pytest.raises(rx.RxGaussError) as e:
        ctx.sync()
    assert e.value.code == rx._lib.RXG_ERR_NOT_SPD
    assert bool((r["status"] == rx._lib.RXG_ERR_NOT_SPD).all())
    ctx.sync()                                                       # reported once
    ok = run(ctx, _stress_model(), y, H=1)                            # the context is clean for the next call
    assert int((ok["status"] != 0).sum()) == 0
