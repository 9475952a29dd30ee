"""Every variant of the shared-model sweep (`lgssm_shared_kernel`, csrc/rxg_lgssm_shared.cuh), chain by chain, against a
plain fp64 Kalman filter + RTS smoother.

The kernel is one template instantiated per (d, m) family x chains per thread (CPT 1 / 2) x smoothing / filtering x
evidence x transition offset x checkpoint-and-recompute (CK: smoothing, d <= 4, CPT 2) x fused peer stores, and each
instantiation meets `transition_first`, a shared missing-data pattern, per-chain prior means and three covariance
outputs at run time.  The tests below drive each of them with `force_cpt` / `sweep_variant`, gate EVERY chain (not a
global norm) and assert the relations that hold bit for bit because both sides run the same `__fmaf_rn` sequence per
chain.

The reference (`reference_sweep`) is deliberately textbook and independent of the library and of the oracle's
message schedule: the chain-independent covariance side runs once in numpy fp64 on the host, the mean side is a
batched torch fp64 recursion on the device the data lives on.  The CPU tests validate it against the oracle to 1e-10.
"""
import itertools

import numpy as np
import pytest
import torch

from oracle import lgssm
from util import TOL_COV, TOL_MEAN, TOL_NLE, f32_model

LOG2PI = float(np.log(2.0 * np.pi))
NATIVE = [(1, 1), (2, 1), (2, 2), (3, 3), (4, 1), (4, 2), (4, 4), (6, 6)]
# general shapes embedded into a register family (embedding_shape in rxg_lgssm_general.cu)
EMBEDDED = {(3, 2): (3, 3), (4, 3): (4, 4), (5, 3): (6, 6)}
SHAPES = NATIVE + list(EMBEDDED)


def family(d, m):
    return EMBEDDED.get((d, m), (d, m))


def ck_eligible(d, m):
    """Smoothing at CPT = 2 checkpoints and recomputes (instead of stashing) when the family has d * d <= 16."""
    D, _ = family(d, m)
    return D * D <= 16


# ====================================================================================== fp64 reference
def _sym(S):
    return 0.5 * (S + np.swapaxes(S, -1, -2))


def covariance_side(mod, T, tmask=None, transition_first=False):
    """Chain-independent half of the Kalman filter + RTS smoother, numpy fp64 on the host.

    Returns per step: predicted / filtered / smoothed covariances, Kalman gains K_t (0 at missing steps), RTS gains G_t,
    the innovation precision S_t^-1 and the evidence constant 1/2 (m log 2 pi + log det S_t) (0 at missing steps)."""
    A, B, P, Q, S0 = (np.asarray(mod[k], np.float64) for k in ("A", "B", "P", "Q", "S0"))
    d, m = A.shape[0], B.shape[0]
    obs = np.ones(T, bool) if tmask is None else np.asarray(tmask).astype(bool)
    assert obs.shape == (T,)
    Sp = np.zeros((T, d, d)); Sf = np.zeros((T, d, d)); K = np.zeros((T, d, m))
    Sinv = np.zeros((T, m, m)); half = np.zeros(T)
    S = S0.copy()
    I = np.eye(d)
    for t in range(T):
        if t > 0 or transition_first:
            S = _sym(A @ S @ A.T + P)
        Sp[t] = S
        if obs[t]:
            Sn = _sym(B @ S @ B.T + Q)
            Si = _sym(np.linalg.inv(Sn))
            Kt = S @ B.T @ Si
            IKB = I - Kt @ B
            S = _sym(IKB @ S @ IKB.T + Kt @ Q @ Kt.T)          # Joseph form
            K[t], Sinv[t] = Kt, Si
            half[t] = 0.5 * (m * LOG2PI + np.linalg.slogdet(Sn)[1])
        Sf[t] = S
    G = np.zeros((T, d, d)); Ss = Sf.copy()
    for t in range(T - 2, -1, -1):
        G[t] = Sf[t] @ A.T @ np.linalg.inv(Sp[t + 1])
        Ss[t] = _sym(Sf[t] + G[t] @ (Ss[t + 1] - Sp[t + 1]) @ G[t].T)
    return dict(obs=obs, Sp=Sp, Sf=Sf, Ss=Ss, K=K, G=G, Sinv=Sinv, half=half, transition_first=transition_first)


def mean_side(cs, mod, y, *, smooth=True, u=None, mu0=None):
    """Per-chain half: batched fp64 recursion over all chains of y[T, m, batch] on y's device.
    ``mu0[d, batch]`` is a per-chain prior mean (default: the model's m0 for every chain).
    Returns (mean[T, d, batch] -- smoothed, or filtered with ``smooth=False`` --, nle[batch])."""
    dev = y.device
    T, m, nb = y.shape
    t64 = lambda a: torch.as_tensor(np.asarray(a, np.float64), dtype=torch.float64, device=dev)
    A, B = t64(mod["A"]), t64(mod["B"])
    d = A.shape[0]
    uu = t64(np.zeros(d) if u is None else u).reshape(d, 1)
    K, G, Si, half = t64(cs["K"]), t64(cs["G"]), t64(cs["Sinv"]), cs["half"]
    tf = cs["transition_first"]
    mu = (mu0.to(dev, torch.float64) if mu0 is not None else t64(mod["m0"]).reshape(d, 1).expand(d, nb)).clone()
    mean = torch.empty(T, d, nb, dtype=torch.float64, device=dev)
    nle = torch.zeros(nb, dtype=torch.float64, device=dev)
    for t in range(T):
        if t > 0 or tf:
            mu = A @ mu + uu
        if cs["obs"][t]:
            e = y[t].to(torch.float64) - B @ mu
            nle += half[t] + 0.5 * (e * (Si[t] @ e)).sum(0)
            mu = mu + K[t] @ e
        mean[t] = mu
    if smooth:                      # RTS, in place: mean[t+1] is already smoothed when step t is visited
        for t in range(T - 2, -1, -1):
            mean[t] += G[t] @ (mean[t + 1] - (A @ mean[t] + uu))
    return mean, nle


def reference_sweep(mod, y, *, smooth=True, u=None, transition_first=False, tmask=None, mu0=None, cs=None):
    """fp64 Kalman filter (+ RTS smoother) of every chain: dict(mean[T, d, batch], cov[T, d, d], nle[batch])."""
    cs = cs if cs is not None else covariance_side(mod, y.shape[0], tmask, transition_first)
    mean, nle = mean_side(cs, mod, y, smooth=smooth, u=u, mu0=mu0)
    return dict(mean=mean, cov=cs["Ss"] if smooth else cs["Sf"], nle=nle)


# ====================================================================================== models and data
def random_model(d, m, seed):
    """Well-conditioned random model.  Q >= 1.5 I keeps every innovation covariance >= 1.5 I, so each observed step adds
    at least 1/2 m (log 2 pi + log 1.5) > 0 to the negative log-evidence: a per-chain relative gate is meaningful."""
    rng = np.random.default_rng(seed)
    Aq, _ = np.linalg.qr(rng.standard_normal((d, d)))
    L = 0.1 * rng.standard_normal((d, d)); N = 0.3 * rng.standard_normal((m, m))
    return f32_model(dict(A=0.95 * Aq, B=rng.standard_normal((m, d)) / np.sqrt(d), P=0.2 * np.eye(d) + L @ L.T,
                          Q=1.5 * np.eye(m) + N @ N.T, m0=rng.standard_normal(d), S0=5.0 * np.eye(d)))


def simulate(mod, T, batch, seed):
    """y[T, m, batch] fp32 drawn from the model itself (vectorised over chains)."""
    rng = np.random.default_rng(seed)
    A, B = mod["A"], mod["B"]
    d, m = A.shape[0], B.shape[0]
    LP, LQ, L0 = (np.linalg.cholesky(mod[k]) for k in ("P", "Q", "S0"))
    x = mod["m0"][:, None] + L0 @ rng.standard_normal((d, batch))
    y = np.empty((T, m, batch))
    for t in range(T):
        if t > 0:
            x = A @ x + LP @ rng.standard_normal((d, batch))
        y[t] = B @ x + LQ @ rng.standard_normal((m, batch))
    return y.astype(np.float32)


def offset(d, seed):
    return (0.5 * np.random.default_rng(seed).standard_normal(d)).astype(np.float32)


def pattern(T):
    """Shared missing-data pattern: step 0 and the last step missing; from T = 20 on, a 14-step gap across the first
    12-step chunk boundary, and two shorter ones."""
    tm = np.ones(T, np.uint8)
    tm[0] = 0
    tm[-1] = 0
    if T >= 20:
        tm[3:17] = 0
    if T >= 50:
        tm[40] = 0
        tm[44:46] = 0
    return tm


def _kw(mod):
    return dict(A=mod["A"], B=mod["B"], P=mod["P"], Q=mod["Q"], m0=mod["m0"], S0=mod["S0"])


# ====================================================================================== per-chain gates
WORST = {}      # category -> (error, case, chain): the measured per-chain worst cases, printed at the end of the module


def _record(cat, err, case, chain):
    if cat not in WORST or err > WORST[cat][0]:
        WORST[cat] = (err, case, chain)


def per_chain_rel(got, ref):
    """Relative L2 over every axis but the last (the chain axis), per chain, in fp64 (chunked over the leading axis)."""
    got = got.to(ref.device)
    num = torch.zeros(ref.shape[-1], dtype=torch.float64, device=ref.device)
    den = torch.zeros_like(num)
    dims = tuple(range(ref.dim() - 1))
    for t0 in range(0, ref.shape[0], 128):
        g, r = got[t0:t0 + 128].to(torch.float64), ref[t0:t0 + 128].to(torch.float64)
        num += ((g - r) ** 2).sum(dims)
        den += (r ** 2).sum(dims)
    err = num.sqrt() / den.sqrt().clamp_min(1e-300)
    return torch.nan_to_num(err, nan=float("inf"))


def gate_mean(cat, case, got, ref, tol=TOL_MEAN):
    err = per_chain_rel(got, ref)
    b = int(err.argmax()); e = float(err[b])
    _record(cat + " mean", e, case, b)
    assert e < tol, f"{case}: mean relative L2 of chain {b} = {e:.3e} >= {tol:g}"
    return e


def gate_nle(cat, case, got, ref, tol=TOL_NLE):
    ref = ref.to(torch.float64)
    err = (got.to(ref.device, torch.float64) - ref).abs() / ref.abs().clamp_min(1e-3)     # no datum at all: nle = 0
    err = torch.nan_to_num(err, nan=float("inf"))
    b = int(err.argmax()); e = float(err[b])
    _record(cat + " nle", e, case, b)
    assert e < tol, f"{case}: nle relative error of chain {b} = {e:.3e} >= {tol:g}"
    return e


def gate_cov(cat, case, cov, ref_tab, tol=TOL_COV):
    """``cov`` per chain [T, d, d, batch] or the de-duplicated table [T, d, d]: every chain must hold the table bit for bit,
    and the table must meet the relative Frobenius gate."""
    tab = cov[..., 0] if cov.dim() == 4 else cov
    if cov.dim() == 4:
        same = (cov == tab[..., None]).flatten(0, 2).all(0)
        bad = (~same).nonzero()
        assert bad.numel() == 0, f"{case}: covariance of chain {int(bad[0])} differs from chain 0"
    r = torch.as_tensor(ref_tab, dtype=torch.float64)
    g = tab.to("cpu", torch.float64)
    e = float((g - r).norm() / r.norm())
    _record(cat + " cov", e, case, -1)
    assert e < tol, f"{case}: covariance relative Frobenius {e:.3e} >= {tol:g}"
    return e


@pytest.fixture(scope="module", autouse=True)
def _report_worst():
    yield
    if WORST:
        print("\nshared-sweep variants, per-chain worst cases:")
        for cat in sorted(WORST):
            e, case, b = WORST[cat]
            print(f"  {cat:<28s} {e:.3e}  ({case}, chain {b})")


# ====================================================================================== CPU: the reference itself
def _oracle_case(d, m, case):
    mod = random_model(d, m, seed=100 * d + m)
    T, batch = (1, 5) if case == "T1" else (30, 5)
    y = simulate(mod, T, batch, seed=7 * d + m)
    kw = dict(u=None, transition_first=False, tmask=None, mu0=None)
    if case == "offset_tf":
        kw.update(u=offset(d, d + m).astype(np.float64), transition_first=True)
    elif case == "offset":
        kw.update(u=offset(d, d + m).astype(np.float64))
    elif case == "mask":
        tm = pattern(T); tm[10:14] = 0
        kw.update(tmask=tm)
    elif case == "all_missing":
        kw.update(tmask=np.zeros(T, np.uint8), transition_first=True)
    elif case == "mu0":
        kw.update(mu0=np.random.default_rng(d).standard_normal((d, batch)))
    return mod, y, kw


def _rel(a, b):
    a = np.asarray(a, np.float64); b = np.asarray(b, np.float64)
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-300))


@pytest.mark.parametrize("d,m", NATIVE)
@pytest.mark.parametrize("case", ["plain", "offset", "offset_tf", "mask", "all_missing", "mu0", "T1"])
def test_reference_matches_oracle(d, m, case):
    """The fp64 reference of this file against the oracle's message schedule and textbook smoother (1e-10)."""
    mod, y, kw = _oracle_case(d, m, case)
    T, _, batch = y.shape
    omod = dict(mod)
    if kw["mu0"] is not None:
        omod["m0"] = kw["mu0"].T.copy()                     # per chain: [batch, d]
    full = None if kw["tmask"] is None else np.repeat(kw["tmask"][:, None], batch, axis=1)
    sched = lgssm.smooth_reference_schedule(y, **omod, mask=full, u=kw["u"], transition_first=kw["transition_first"])
    rts = lgssm.kalman_rts(y, **omod, mask=full, u=kw["u"], transition_first=kw["transition_first"])
    mu0 = None if kw["mu0"] is None else torch.as_tensor(kw["mu0"])
    yt = torch.as_tensor(y)
    cs = covariance_side(mod, T, kw["tmask"], kw["transition_first"])
    sm = reference_sweep(mod, yt, smooth=True, u=kw["u"], mu0=mu0, cs=cs)
    fl = reference_sweep(mod, yt, smooth=False, u=kw["u"], mu0=mu0, cs=cs)
    for ref in (sched, rts):
        assert _rel(sm["mean"].numpy(), ref["mean"]) < 1e-10
        assert _rel(fl["mean"].numpy(), ref["filt_mean"]) < 1e-10
        assert _rel(np.broadcast_to(cs["Ss"][..., None], ref["cov"].shape), ref["cov"]) < 1e-10
        assert _rel(np.broadcast_to(cs["Sf"][..., None], ref["filt_cov"].shape), ref["filt_cov"]) < 1e-10
        for got in (sm["nle"].numpy(), fl["nle"].numpy()):
            assert np.all(np.abs(got - ref["neg_log_evidence"]) <= 1e-10 * np.maximum(1.0, np.abs(ref["neg_log_evidence"])))
    if kw["tmask"] is not None and not kw["tmask"].any():
        assert np.all(sm["nle"].numpy() == 0.0)


@pytest.mark.parametrize("d,m", NATIVE)
def test_reference_matches_streaming_oracle(d, m):
    """Filtering with the prior one transition before the first datum = the oracle's streaming filter, also with a
    per-chain prior mean and a prior covariance other than S0 (the streaming engine's carry)."""
    mod = random_model(d, m, seed=300 + 10 * d + m)
    y = simulate(mod, 25, 6, seed=d + 2 * m)
    rng = np.random.default_rng(d * m)
    mu0 = rng.standard_normal((d, 6))
    C = rng.standard_normal((d, d))
    mod2 = dict(mod, S0=np.asarray(2.0 * np.eye(d) + 0.2 * C @ C.T, np.float32).astype(np.float64))
    u = offset(d, 5).astype(np.float64)
    ref = lgssm.filter_streaming(y, **dict(mod2, m0=mu0.T.copy()), u=u)
    r = reference_sweep(mod2, torch.as_tensor(y), smooth=False, u=u, transition_first=True, mu0=torch.as_tensor(mu0))
    assert _rel(r["mean"].numpy(), ref["mean"]) < 1e-10
    assert _rel(np.broadcast_to(r["cov"][..., None], ref["cov"].shape), ref["cov"]) < 1e-10


def test_pattern_has_the_edges_the_matrix_needs():
    for T in (1, 5, 12, 13, 25, 65):
        tm = pattern(T)
        assert tm[0] == 0 and tm[-1] == 0
    runs = np.diff(np.flatnonzero(np.diff(np.r_[1, pattern(65), 1])))[::2]
    assert runs.max() > 12


# ====================================================================================== GPU: the variant matrix
OPTIONS = list(itertools.product((True, False), (False, True), (False, True), (False, True), (False, True)))
COV_MODES = ("chain", "shared", "none")
MATRIX_T = [1, 5, 12, 13, 25, 65]
SWEEP_T = [1, 2, 3, 4, 5, 11, 12, 13, 16, 17, 24, 25, 63, 64, 65, 128, 129]


def _sweep(ctx, y, mod, *, cpt, variant, smooth=True, evid=False, u=None, tf=False, tm=None, cov_mode="chain", **kw):
    ctx.set_option("force_cpt", cpt)
    ctx.set_option("sweep_variant", variant)
    return ctx.lgssm(y, **_kw(mod), u=u, smooth=smooth, mask=tm, want_cov=cov_mode != "none", want_evidence=evid,
                     cov_shared_out=cov_mode == "shared", transition_first=tf, **kw)


def _eq(a, b, what, case):
    if a is None and b is None:
        return
    assert a is not None and b is not None and torch.equal(a, b), f"{case}: {what} not bit-identical"


def _check(cat, case, r, ref, nb, *, evid, cov_mode):
    gate_mean(cat, case, r["mean"], ref["mean"][..., :nb])
    if evid:
        gate_nle(cat, case, r["neg_log_evidence"], ref["nle"][:nb])
    if cov_mode != "none":
        gate_cov(cat, case, r["cov"], ref["cov"])
    else:
        assert r["cov"] is None


@pytest.mark.gpu
@pytest.mark.parametrize("T", MATRIX_T)
@pytest.mark.parametrize("d,m", SHAPES)
def test_variant_matrix(ctx, d, m, T):
    """All options x CPT 1 / 2 x stash / CK at batch 70 (ragged: the second CPT = 2 CTA has 3 live lanes), 2 (one CPT = 2
    pair) and 71 (odd: CPT = 2 requested, CPT = 1 taken), every chain gated, exact relations asserted."""
    mod = random_model(d, m, seed=1000 + 16 * d + m)
    u_vec = offset(d, 17 * d + m)
    y_np = simulate(mod, T, 71, seed=31 * T + d + m)
    tm = pattern(T)
    y_mask_np = y_np.copy()
    y_mask_np[tm == 0] = 1.0e3               # values at missing steps must not reach any output
    ck = ck_eligible(d, m)
    cs_cache = {}
    for i, (smooth, evid, use_u, tf, use_mask) in enumerate(OPTIONS):
        cov_mode = COV_MODES[i % 3]
        case = (f"d={d} m={m} T={T} {'smooth' if smooth else 'filter'} evid={int(evid)} u={int(use_u)} tf={int(tf)} "
                f"mask={int(use_mask)} cov={cov_mode}")
        u = u_vec if use_u else None
        tmk = tm if use_mask else None
        y71 = torch.as_tensor(y_mask_np if use_mask else y_np, device="cuda")
        key = (use_mask, tf)
        if key not in cs_cache:
            cs_cache[key] = covariance_side(mod, T, tmk, tf)
        ref = reference_sweep(mod, y71.cpu(), smooth=smooth, u=None if u is None else u.astype(np.float64), cs=cs_cache[key])
        y70 = y71[..., :70].contiguous()
        kw = dict(smooth=smooth, evid=evid, u=u, tf=tf, tm=tmk, cov_mode=cov_mode)
        cat = "matrix"
        r1 = _sweep(ctx, y70, mod, cpt=1, variant=0, **kw)
        _check(cat, case + " cpt=1", r1, ref, 70, evid=evid, cov_mode=cov_mode)
        r2 = _sweep(ctx, y70, mod, cpt=2, variant=0, **kw)               # CK when smoothing at d <= 4
        _check(cat, case + " cpt=2", r2, ref, 70, evid=evid, cov_mode=cov_mode)
        rs = r2
        if smooth and ck:
            rs = _sweep(ctx, y70, mod, cpt=2, variant=1, **kw)           # the stash at CPT = 2
            _check(cat, case + " cpt=2 stash", rs, ref, 70, evid=evid, cov_mode=cov_mode)
        # ---- exact relations
        if not evid:
            for r in (r2, rs):
                _eq(r1["mean"], r["mean"], "mean across CPT / stash / CK", case)
                _eq(r1["cov"], r["cov"], "cov across CPT / stash / CK", case)
        if not smooth:
            _eq(r1["mean"], r2["mean"], "filtered mean across CPT", case)
        if evid:
            _eq(r1["neg_log_evidence"], r2["neg_log_evidence"], "nle across CPT", case)
            _eq(r1["neg_log_evidence"], rs["neg_log_evidence"], "nle across stash / CK", case)
        if cov_mode != "none":
            _eq(r1["cov"], r2["cov"], "covariances across CPT", case)
        # chain order reversed: chains change lanes, pair slots and CTAs
        rr = _sweep(ctx, y70.flip(-1).contiguous(), mod, cpt=2, variant=0, **kw)
        _eq(rr["mean"].flip(-1), r2["mean"], "mean under chain reversal", case)
        if evid:
            _eq(rr["neg_log_evidence"].flip(-1), r2["neg_log_evidence"], "nle under chain reversal", case)
        if cov_mode == "chain":
            rt = _sweep(ctx, y70, mod, cpt=2, variant=0, **dict(kw, cov_mode="shared"))
            assert torch.equal(r2["cov"], rt["cov"][..., None].expand_as(r2["cov"])), f"{case}: per-chain cov != shared table"
            _eq(rt["mean"], r2["mean"], "mean with / without the shared covariance table", case)
        # ---- one CPT = 2 pair: both lanes of the pair, same bits as inside the larger batch
        for variant in ((0, 1) if smooth and ck else (0,)):
            rp = _sweep(ctx, y70[..., :2].contiguous(), mod, cpt=2, variant=variant, **kw)
            _check(cat, case + f" batch=2 v={variant}", rp, ref, 2, evid=evid, cov_mode=cov_mode)
            rb = r2 if variant == 0 else rs
            _eq(rp["mean"], rb["mean"][..., :2], "batch-2 mean vs batch-70 mean", case)
        # ---- odd batch with CPT = 2 requested: the CPT = 1 kernel runs
        ro = _sweep(ctx, y71, mod, cpt=2, variant=0, **kw)
        _check(cat, case + " batch=71", ro, ref, 71, evid=evid, cov_mode=cov_mode)
        _eq(ro["mean"][..., :70], r1["mean"], "odd batch (CPT = 1 fallback) vs CPT = 1", case)
        if evid:
            _eq(ro["neg_log_evidence"][:70], r1["neg_log_evidence"], "odd batch nle vs CPT = 1", case)


@pytest.mark.gpu
@pytest.mark.parametrize("d,m", SHAPES)
def test_smoothing_over_chunk_boundaries(ctx, d, m):
    """The plain smoothing call, with and without evidence, at both CPT over T around the PF = 4 prefetch, the 12-step
    (CK) / 16-step table chunks and the 64-step fp64 flush of the evidence; CK + evidence + offset (with and without
    transition_first) at every T."""
    mod = random_model(d, m, seed=2000 + 16 * d + m)
    u = offset(d, 3 * d + m)
    ck = ck_eligible(d, m)
    for T in SWEEP_T:
        y = torch.as_tensor(simulate(mod, T, 70, seed=7 * T + d * m), device="cuda")
        yc = y.cpu()
        cs = covariance_side(mod, T)
        ref = reference_sweep(mod, yc, cs=cs)
        for evid in (False, True):
            case = f"d={d} m={m} T={T} evid={int(evid)}"
            outs = []
            for cpt, variant in ((1, 0), (2, 0)) + (((2, 1),) if ck else ()):
                r = _sweep(ctx, y, mod, cpt=cpt, variant=variant, evid=evid)
                _check("T sweep", case + f" cpt={cpt} v={variant}", r, ref, 70, evid=evid, cov_mode="chain")
                outs.append(r)
            for r in outs[1:]:
                if not evid:
                    _eq(outs[0]["mean"], r["mean"], "mean across CPT / stash / CK", case)
                else:
                    _eq(outs[0]["neg_log_evidence"], r["neg_log_evidence"], "nle across CPT / stash / CK", case)
                _eq(outs[0]["cov"], r["cov"], "cov across CPT / stash / CK", case)
        for tf in (False, True):          # CK (d <= 4) + EVID + OFFSET, prior on x[1] or one transition earlier
            case = f"d={d} m={m} T={T} evid=1 u=1 tf={int(tf)}"
            refu = reference_sweep(mod, yc, u=u.astype(np.float64), transition_first=tf)
            r = _sweep(ctx, y, mod, cpt=2, variant=0, evid=True, u=u, tf=tf)
            _check("T sweep", case, r, refu, 70, evid=True, cov_mode="chain")
            rf = _sweep(ctx, y, mod, cpt=2, variant=0, smooth=False, evid=True, u=u, tf=tf, cov_mode="none")
            gate_mean("T sweep filter", case, rf["mean"], reference_sweep(mod, yc, smooth=False, u=u.astype(np.float64),
                                                                          transition_first=tf)["mean"])
            _eq(rf["neg_log_evidence"], r["neg_log_evidence"], "nle filter vs smoother", case)


@pytest.mark.gpu
@pytest.mark.parametrize("d,m", SHAPES)
def test_streaming_chunk_per_chain_prior(ctx, d, m):
    """`lgssm_filter_chunk` (the streaming engine's chunk): a random per-chain prior mean `prev_mean` (mu0c in the
    kernel) and a carried prior covariance, at both CPT, against the reference run with that prior."""
    mod = random_model(d, m, seed=3000 + 16 * d + m)
    T, nb = 29, 70
    rng = np.random.default_rng(d * 10 + m)
    y = torch.as_tensor(simulate(mod, T, nb, seed=d + m), device="cuda")
    prev = torch.as_tensor(rng.standard_normal((d, nb)).astype(np.float32), device="cuda")
    C = rng.standard_normal((d, d))
    carry0 = np.asarray(2.0 * np.eye(d) + 0.2 * C @ C.T, np.float32)
    cmod = dict(mod, S0=carry0.astype(np.float64))
    u = offset(d, m)
    for evid, use_u in itertools.product((False, True), (False, True)):
        uu = u if use_u else None
        ref = reference_sweep(cmod, y.cpu(), smooth=False, u=None if uu is None else uu.astype(np.float64),
                              transition_first=True, mu0=prev.cpu())
        outs = []
        for cpt in (1, 2):
            case = f"d={d} m={m} evid={int(evid)} u={int(use_u)} cpt={cpt}"
            ctx.set_option("force_cpt", cpt)
            cc = carry0.copy()
            r = ctx.lgssm_filter_chunk(y, mod["A"], mod["B"], mod["P"], mod["Q"], prev, cc, u=uu, want_evidence=evid)
            gate_mean("streaming", case, r["mean"], ref["mean"])
            if evid:
                gate_nle("streaming", case, r["neg_log_evidence"], ref["nle"])
            gate_cov("streaming", case, r["cov"], ref["cov"])
            np.testing.assert_array_equal(cc, r["cov"][-1, :, :, 0].cpu().numpy())     # the carry out
            outs.append(r)
            rr = ctx.lgssm_filter_chunk(y.flip(-1).contiguous(), mod["A"], mod["B"], mod["P"], mod["Q"],
                                        prev.flip(-1).contiguous(), carry0.copy(), u=uu, want_evidence=evid)
            _eq(rr["mean"].flip(-1), r["mean"], "streaming mean under chain reversal", case)
        _eq(outs[0]["mean"], outs[1]["mean"], "streaming mean across CPT", case)
        if evid:
            _eq(outs[0]["neg_log_evidence"], outs[1]["neg_log_evidence"], "streaming nle across CPT", case)


@pytest.mark.gpu
@pytest.mark.parametrize("d,m", [(4, 4), (3, 3), (6, 6)])
def test_misaligned_caller_buffers_fall_back_to_one_chain_per_thread(ctx, d, m):
    """Caller buffers that are not 16-byte aligned (4-byte storage offset) with CPT = 2 requested: the CPT = 1 kernel
    runs, bit-identical to aligned buffers at CPT = 1."""
    mod = random_model(d, m, seed=4000 + d)
    T, nb = 37, 70
    y = torch.as_tensor(simulate(mod, T, nb, seed=d), device="cuda")
    u = offset(d, 1)

    def off4(*shape):
        n = int(np.prod(shape))
        t = torch.empty(n + 1, device="cuda")[1:].view(*shape)
        assert t.data_ptr() % 16 == 4 and t.is_contiguous()
        return t

    y_mis = off4(T, m, nb).copy_(y)
    for smooth in (True, False):
        kw = dict(smooth=smooth, evid=True, u=u, tf=smooth)
        case = f"d={d} m={m} {'smooth' if smooth else 'filter'}"
        base = _sweep(ctx, y, mod, cpt=1, variant=0, **kw)
        for what, extra, yy in (("out_mean", dict(out_mean=off4(T, d, nb)), y),
                                ("out_cov", dict(out_cov=off4(T, d, d, nb)), y),
                                ("y", {}, y_mis)):
            r = _sweep(ctx, yy, mod, cpt=2, variant=0, **kw, **extra)
            _eq(r["mean"], base["mean"], f"mean with misaligned {what}", case)
            _eq(r["cov"], base["cov"], f"cov with misaligned {what}", case)
            _eq(r["neg_log_evidence"], base["neg_log_evidence"], f"nle with misaligned {what}", case)
        ref = reference_sweep(mod, y.cpu(), smooth=smooth, u=u.astype(np.float64), transition_first=smooth)
        _check("misaligned", case, base, ref, nb, evid=True, cov_mode="chain")


# ====================================================================================== GPU: full size, every chain
FULL_T, FULL_B = 1000, 65536


@pytest.fixture(scope="module")
def full_y():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    g = torch.Generator(device="cuda").manual_seed(4242)
    y = torch.randn(FULL_T, 4, FULL_B, device="cuda", generator=g) * 3.3     # bench.py's data
    yield y
    del y
    torch.cuda.empty_cache()


def _full_case(ctx, full_y, *, smooth=True, evid=False, u=None, tf=False, tm=None, reverse=False):
    mod = f32_model(lgssm.notebook_model(4))
    case = f"full size {'smooth' if smooth else 'filter'} evid={int(evid)} u={int(u is not None)} tf={int(tf)} mask={int(tm is not None)}"
    r = ctx.lgssm(full_y, **_kw(mod), u=u, smooth=smooth, mask=tm, want_evidence=evid, transition_first=tf)
    ref = reference_sweep(mod, full_y, smooth=smooth, u=None if u is None else u.astype(np.float64), transition_first=tf,
                          tmask=tm)
    em = gate_mean("full", case, r["mean"], ref["mean"])
    en = gate_nle("full", case, r["neg_log_evidence"], ref["nle"]) if evid else None
    ec = gate_cov("full", case, r["cov"], ref["cov"])
    print(f"{case}: worst chain mean {em:.2e}, cov {ec:.2e}" + (f", nle {en:.2e}" if evid else ""))
    del ref
    if reverse:
        rr = ctx.lgssm(full_y.flip(-1).contiguous(), **_kw(mod), u=u, smooth=smooth, mask=tm, want_evidence=evid,
                       transition_first=tf)
        assert torch.equal(rr["mean"].flip(-1), r["mean"])
        assert torch.equal(rr["cov"], r["cov"])            # chain independent
        del rr
    del r
    torch.cuda.empty_cache()


@pytest.mark.gpu
def test_full_size_benchmarked_call_every_chain(ctx, full_y):
    """bench.py's call (notebook model, d = m = 4, T = 1000, 65 536 chains, default dispatch = CPT 2 + CK): all chains
    against the fp64 reference, and the reversed batch bit for bit."""
    _full_case(ctx, full_y, reverse=True)


@pytest.mark.gpu
@pytest.mark.parametrize("variant", ["evidence", "offset_tf", "mask", "filter_evidence"])
def test_full_size_variants_every_chain(ctx, full_y, variant):
    kw = dict(evidence=dict(evid=True),
              offset_tf=dict(u=offset(4, 99), tf=True),
              mask=dict(tm=pattern(FULL_T), evid=True),
              filter_evidence=dict(smooth=False, evid=True))[variant]
    _full_case(ctx, full_y, **kw)


@pytest.mark.gpu
def test_outputs_beyond_2_pow_31_elements(ctx):
    """d = 4, T = 1000, 135 000 chains: 2.16e9 covariance elements (> 2^31) and ~13 GB of outputs."""
    T, nb = 1000, 135000
    need = 4 * T * nb * (4 + 4 + 16) + (2 << 30)
    free, _ = torch.cuda.mem_get_info()
    if free < need:
        pytest.skip(f"needs {need / 2**30:.1f} GiB of free device memory, {free / 2**30:.1f} GiB free (shared device)")
    assert T * 16 * nb > 2 ** 31
    mod = f32_model(lgssm.notebook_model(4))
    g = torch.Generator(device="cuda").manual_seed(99)
    y = torch.randn(T, 4, nb, device="cuda", generator=g) * 3.3
    r = ctx.lgssm(y, **_kw(mod), smooth=True, want_evidence=True)
    mean, cov, nle = r["mean"], r["cov"], r["neg_log_evidence"]
    del r
    idx = torch.cat([torch.arange(0, 64), torch.arange(nb // 2 - 32, nb // 2 + 32), torch.arange(nb - 64, nb)]).cuda()
    ref = reference_sweep(mod, y[..., idx].contiguous())
    del y
    gate_mean("beyond 2^31", "135000 chains", mean[..., idx], ref["mean"])
    gate_nle("beyond 2^31", "135000 chains", nle[idx], ref["nle"])
    last = cov[..., nb - 1].clone()
    assert torch.equal(last, cov[..., 0])
    gate_cov("beyond 2^31", "135000 chains, last chain", last, ref["cov"])
    del mean, cov, nle
    torch.cuda.empty_cache()


# ====================================================================================== GPU: fused peer stores at CPT = 2
class _quiet_host:
    """Virtual ranks share one process: while one rank's barrier kernel spins, the host must not run anything that
    synchronises the whole device (the cyclic GC freeing device buffers) before the other ranks' work is queued."""

    def __enter__(self):
        import gc
        gc.collect()
        torch.cuda.synchronize()
        gc.disable()

    def __exit__(self, *a):
        import gc
        gc.enable()


@pytest.fixture(scope="module")
def ranks(rx):
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    cs = [rx.Context(0, use_torch_stream=False) for _ in range(3)]
    yield cs
    for c in cs:
        c.close()


@pytest.mark.gpu
@pytest.mark.parametrize("G", [2, 3])
@pytest.mark.parametrize("variant", ["full", "replicate"])
def test_peer_fused_gather_two_chains_per_thread(rx, ranks, G, variant):
    """The PEER + CK + CPT = 2 instantiation (what bench.py runs at N > 1), on virtual ranks: gathered buffers bit-identical
    to per-shard sweeps at the same CPT, every chain gated against the reference."""
    from rxinfer_jl_b200.sharding import PeerGroup
    mod = f32_model(lgssm.notebook_model(4))
    T, b = 61, 70                                     # 70 chains per shard: ragged second CTA at CPT = 2
    cs = ranks[:G]
    try:
        for c in cs:                                  # module-scoped contexts: set and reset their options here
            c.set_option("gather_mode", 0)
            c.set_option("force_cpt", 2)
            c.set_option("sweep_variant", 0)
        y = torch.as_tensor(simulate(mod, T, G * b, seed=G), device="cuda")
        groups = PeerGroup.local(cs, T, 4, b)
        refs = []
        for r, c in enumerate(cs):                    # per-shard sweeps (also load every kernel before any barrier spins)
            ys = y[..., r * b:(r + 1) * b].contiguous()
            refs.append((ys, c.lgssm(ys, **_kw(mod), smooth=True)))
        for gr in groups:
            gr.mean.zero_(); gr.cov.zero_()
        torch.cuda.synchronize()
        with _quiet_host():
            for r, gr in enumerate(groups):
                gr.smooth_gather(refs[r][0], mod, replicate_cov=(variant == "replicate"), asynchronous=True)
            for c in cs:
                c.sync()
        for gr in groups:
            for r in range(G):
                assert torch.equal(gr.mean[r], refs[r][1]["mean"]), (variant, gr.rank, r)
                assert torch.equal(gr.cov[r], refs[r][1]["cov"]), (variant, gr.rank, r)
        full = rx.sharding.assemble_gathered(groups[0].mean)
        ref = reference_sweep(mod, y.cpu())
        gate_mean("peer", f"G={G} {variant}", full, ref["mean"])
        gate_cov("peer", f"G={G} {variant}", rx.sharding.assemble_gathered(groups[0].cov), ref["cov"])
    finally:
        for c in cs:
            c.set_option("force_cpt", 0)
            c.set_option("gather_mode", 0)
            c.set_option("sweep_variant", 0)
