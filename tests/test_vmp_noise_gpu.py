"""rxg_lgssm_vmp_noise_f32 on the GPU: every chain gated against the fp64 reference of test_vmp_noise.py at the unchanged
TOL_MEAN / TOL_COV (q(x), relative L2 / Frobenius per chain), TOL_COV for the inverse scales of q(w_p) and q(w_q) at every
iteration (relative Frobenius per chain), df exactly and the free energy at TOL_NLE (relative to max(|F|, 1), per chain
and iteration); bit-exact relations with torch.equal; the full-size call; the refusals of the C entry."""
import ctypes
from ctypes import c_void_p

import numpy as np
import pytest
import torch

from test_vmp_noise import lgssm_wishart_noise, p_prior, q_prior
from test_vmp_wishart import random_problem
from test_vmp_wishart_gpu import _per_chain_rel, monotone
from util import TOL_COV, TOL_MEAN, TOL_NLE

SHAPES = [(1, 1), (2, 1), (2, 2), (2, 3), (3, 3), (4, 2), (4, 4), (5, 3), (6, 6)]
NB = 7                                                   # odd batch
f32 = lambda M: np.asarray(M, np.float32).astype(np.float64)


def learn_kwargs(mod, learn, d, m, p_init=None, q_init=None):
    """Arguments (fp32-exact) for learn = "P", "PQ" or "Q": learned noises get their prior and initial E[w]."""
    kw = {}
    if "P" in learn:
        nu, S = p_prior(d)
        kw.update(p_prior=(nu, f32(S)), p_init=f32(np.linalg.inv(mod["P"]) if p_init is None else p_init))
    else:
        kw["P"] = mod["P"]
    if "Q" in learn:
        nu, S = q_prior(m)
        kw.update(q_prior=(nu, f32(S)), q_init=f32(np.eye(m) * 1.5 if q_init is None else q_init))
    else:
        kw["Q"] = f32(np.eye(m) * 0.5)
    return kw


def gate(case, r, ref):
    mean, cov = r["mean"].cpu().numpy(), r["cov"].cpu().numpy()
    em = _per_chain_rel(mean, ref["mean"], (0, 1)); ec = _per_chain_rel(cov, ref["cov"], (0, 1, 2))
    assert em.max() <= TOL_MEAN, f"{case}: q(x) mean rel L2 {em.max():.3g} (chain {em.argmax()})"
    assert ec.max() <= TOL_COV, f"{case}: q(x) cov rel Frobenius {ec.max():.3g} (chain {ec.argmax()})"
    for w in ("p", "q"):
        if f"df_{w}" not in ref:
            assert r[f"df_{w}"] is None and r[f"inv_scale_{w}"] is None, case
            continue
        assert np.array_equal(r[f"df_{w}"].cpu().numpy().astype(np.float64), ref[f"df_{w}"]), f"{case}: df_{w}"
        ep = _per_chain_rel(r[f"inv_scale_{w}"].cpu().numpy(), ref[f"inv_scale_{w}"], (1, 2))
        assert ep.max() <= TOL_COV, f"{case}: inv_scale_{w} rel Frobenius {ep.max():.3g} at {np.unravel_index(ep.argmax(), ep.shape)}"
    if r["free_energy"] is not None:
        fe = r["free_energy"].cpu().numpy()
        ef = np.abs(fe - ref["free_energy"]) / np.maximum(np.abs(ref["free_energy"]), 1.0)
        assert ef.max() <= TOL_NLE, f"{case}: free energy rel {ef.max():.3g} at {np.unravel_index(ef.argmax(), ef.shape)}"


def _mask(kind, T):
    if kind == "chain":
        mk = np.ones((T, NB), dtype=np.uint8)
        mk[max(T - 3, 0):, 1] = 0                    # trailing gap
        mk[0, 2] = 0
        mk[T // 2, 3] = 0
        mk[:, 4] = 0                                  # all missing
        return mk
    if kind == "shared":
        mk = np.ones(T, dtype=np.uint8)
        mk[T - 1] = 0
        if T > 2:
            mk[1] = 0
        return mk
    return None


def run(ctx, mod, y, its, kw, *, mask=None, u=None, tf=False, fe=True):
    mk = None if mask is None else (torch.as_tensor(mask, device="cuda") if mask.ndim == 2 else mask)
    r = ctx.lgssm_vmp_noise(torch.as_tensor(y, device="cuda"), mod["A"], mod["B"], mod["m0"], mod["S0"], **kw,
                            iterations=its, u=u, mask=mk, transition_first=tf, want_free_energy=fe)
    torch.cuda.synchronize()
    return r


# (iterations, mask, transition_first, constant u) per row: every (d, m, T, learn) runs all three
VARIANTS = [(1, None, False, False), (5, "chain", True, True), (20, "shared", False, True)]


@pytest.mark.gpu
@pytest.mark.parametrize("learn", ["P", "PQ"])
@pytest.mark.parametrize("T", [1, 2, 37, 300])
@pytest.mark.parametrize("d,m", SHAPES)
def test_matrix(ctx, d, m, T, learn):
    mod, y, _, _ = random_problem(d, m, T, NB, seed=100 * d + 10 * m + T)
    kw = learn_kwargs(mod, learn, d, m)
    for its, mk, tf, with_u in VARIANTS:
        case = f"learn={learn} d={d} m={m} T={T} its={its} mask={mk} tf={int(tf)} u={int(with_u)}"
        u = f32(np.linspace(-0.2, 0.3, d)) if with_u else None
        mask = _mask(mk, T)
        r = run(ctx, mod, y, its, kw, mask=mask, u=u, tf=tf)
        assert int(r["status"].abs().sum()) == 0, f"{case}: status {r['status'].tolist()}"
        ref = lgssm_wishart_noise(y, mod["A"], mod["B"], mod["m0"], mod["S0"], its, mask=mask, u=u, transition_first=tf,
                                  **kw)
        gate(case, r, ref)
        monotone(r["free_energy"], case)


@pytest.mark.gpu
@pytest.mark.parametrize("d,m", [(1, 1), (2, 3), (4, 4), (5, 3), (6, 6)])
def test_learn_q_equals_the_observation_precision_entry(ctx, d, m):
    """Q learned and P known through rxg_lgssm_vmp_noise_f32 equals rxg_lgssm_vmp_wishart_f32 on every output."""
    T, its = 40, 5
    mod, y, _, _ = random_problem(d, m, T, NB, seed=3 * d + m)
    mask = _mask("chain", T)
    u = f32(np.linspace(-0.1, 0.2, d))
    yy, mk = torch.as_tensor(y, device="cuda"), torch.as_tensor(mask, device="cuda")
    nu0, Psi0 = q_prior(m)
    a = ctx.lgssm_vmp_wishart(yy, mod["A"], mod["B"], mod["P"], mod["m0"], mod["S0"], iterations=its, w_prior=(nu0, Psi0),
                              init_E_W=np.eye(m) * 1.5, u=u, mask=mk, transition_first=True, want_free_energy=True)
    b = ctx.lgssm_vmp_noise(yy, mod["A"], mod["B"], mod["m0"], mod["S0"], P=mod["P"], q_prior=(nu0, Psi0),
                            q_init=np.eye(m) * 1.5, u=u, mask=mk, transition_first=True, iterations=its,
                            want_free_energy=True)
    torch.cuda.synchronize()
    for ka, kb in (("mean", "mean"), ("cov", "cov"), ("df", "df_q"), ("inv_scale", "inv_scale_q"),
                   ("free_energy", "free_energy"), ("status", "status")):
        assert torch.equal(a[ka], b[kb]), ka
    assert b["df_p"] is None and b["inv_scale_p"] is None


@pytest.mark.gpu
@pytest.mark.parametrize("d,m", [(2, 2), (3, 3), (4, 4), (4, 2)])
def test_one_iteration_is_the_per_chain_smoother(ctx, d, m):
    """Learn-P at iterations = 1 with init_E_Wp = inv(P), P diagonal with power-of-two entries (the fp64 inversion gives P
    back exactly in fp32): q(x) equals Context.lgssm(..., force_per_chain_path=True), bit for bit -- both kernels run the
    same step helpers, and the pair hook only reads the RTS step's values."""
    T = 40
    mod, y, _, _ = random_problem(d, m, T, NB, seed=9 * d + m)
    P = np.diag([0.5, 2.0, 0.25, 1.0, 4.0, 0.125][:d])
    Q = np.diag([0.5, 0.25, 1.0, 2.0][:m])
    mask = _mask("chain", T)
    yy = torch.as_tensor(y, device="cuda")
    for tf, u, mk in ((False, None, None), (True, np.linspace(-0.1, 0.2, d), mask)):
        kw = dict(Q=Q, p_prior=(d + 2.0, np.eye(d)), p_init=np.linalg.inv(P))
        r = run(ctx, mod, y, 1, kw, mask=mk, u=u, tf=tf, fe=False)
        ref = ctx.lgssm(yy, mod["A"], mod["B"], P, Q, mod["m0"], mod["S0"], u=u, smooth=True, force_per_chain_path=True,
                        mask=None if mk is None else torch.as_tensor(mk, device="cuda"), transition_first=tf)
        assert torch.equal(r["mean"], ref["mean"]) and torch.equal(r["cov"], ref["cov"]), (tf, mk is not None)


@pytest.mark.gpu
@pytest.mark.parametrize("learn", ["P", "PQ"])
@pytest.mark.parametrize("d,m", [(2, 2), (3, 3), (4, 4), (5, 3)])
def test_exact_relations(ctx, d, m, learn):
    """A reversed batch gives the reversed results, a chain run alone equals the same chain inside the batch
    (torch.equal)."""
    T, its = 50, 6
    mod, y, _, _ = random_problem(d, m, T, NB, seed=5 * d + m)
    kw = learn_kwargs(mod, learn, d, m)
    mask = _mask("chain", T)
    keys = ["mean", "cov", "free_energy", "df_p", "inv_scale_p"] + (["df_q", "inv_scale_q"] if "Q" in learn else [])
    r = run(ctx, mod, y, its, kw, mask=mask, tf=True)
    rr = run(ctx, mod, np.ascontiguousarray(y[..., ::-1]), its, kw, mask=np.ascontiguousarray(mask[:, ::-1]), tf=True)
    for k in keys + ["status"]:
        assert torch.equal(rr[k].flip(-1), r[k]), k
    for c in (0, 3, NB - 1):
        r1 = run(ctx, mod, np.ascontiguousarray(y[..., c:c + 1]), its, kw, mask=np.ascontiguousarray(mask[:, c:c + 1]),
                 tf=True)
        for k in keys:
            assert torch.equal(r1[k][..., 0], r[k][..., c]), (k, c)


@pytest.mark.gpu
def test_full_size(ctx):
    """d = m = 4, T = 1000, 65 536 chains, 10 iterations, both precisions learned: every status OK, the free energy
    monotone for every chain, and 64 sampled chains (both ends and the middle) against the reference."""
    d, m, T, nb, its = 4, 4, 1000, 65536, 10
    mod, y8, _, _ = random_problem(d, m, T, 64, seed=4)
    rng = np.random.default_rng(5)
    y = torch.as_tensor(y8, device="cuda").repeat(1, 1, nb // 64)
    y += torch.as_tensor(rng.standard_normal((1, m, nb)).astype(np.float32) * 0.3, device="cuda")
    kw = learn_kwargs(mod, "PQ", d, m)
    r = ctx.lgssm_vmp_noise(y, mod["A"], mod["B"], mod["m0"], mod["S0"], **kw, iterations=its, want_free_energy=True)
    torch.cuda.synchronize()
    assert int((r["status"] != 0).sum()) == 0
    monotone(r["free_energy"], "full size")
    idx = np.r_[0:22, nb // 2 - 10:nb // 2 + 10, nb - 22:nb]
    ys = y[..., idx].cpu().numpy()
    ref = lgssm_wishart_noise(ys, mod["A"], mod["B"], mod["m0"], mod["S0"], its, **kw)
    sub = {k: (v[..., idx] if v is not None else None) for k, v in r.items() if k != "status"}
    gate("full size", sub, ref)


# ====================================================================================== refusals
def _raw(ctx, d=2, m=2, T=4, nb=3, its=2, flags=None, learn="PQ", nu_p=4.0, nu_q=4.0, iSp=None, EWp=None, iSq=None,
         EWq=None, P=None, Q=None, outs=None, dev=True):
    """One raw call of the export; learn says which pairs / outputs are passed, the keywords override single arguments
    (the string "none" passes NULL)."""
    from rxinfer_jl_b200 import _lib as L
    keep = []

    def hp(a, shape):
        if isinstance(a, str):
            return L.as_fp(0)
        a = np.ascontiguousarray(np.eye(shape, dtype=np.float32) if a is None else np.asarray(a, np.float32))
        keep.append(a)
        return a.ctypes.data_as(L.fp)
    A = np.eye(d, dtype=np.float32); B = np.ones((m, d), np.float32)
    m0 = np.zeros(d, np.float32); S0 = np.eye(d, dtype=np.float32)
    mm, dd, ii = max(m, 1), max(d, 1), max(its, 1)
    mk = (lambda *s: torch.empty(*s, device="cuda")) if dev else (lambda *s: torch.empty(*s))
    y = torch.zeros(T, mm, nb, device="cuda" if dev else "cpu")
    mean, cov = mk(T, dd, nb), mk(T, dd, dd, nb)
    o = dict(df_p=mk(ii, nb), iS_p=mk(ii, dd, dd, nb), df_q=mk(ii, nb), iS_q=mk(ii, mm, mm, nb))
    lp, lq = "P" in learn, "Q" in learn
    use = dict(df_p=lp, iS_p=lp, df_q=lq, iS_q=lq)
    use.update(outs or {})
    p = lambda t: L.as_fp(t.data_ptr())
    op = {k: (p(v) if use[k] else L.as_fp(0)) for k, v in o.items()}
    args_p = ((hp("none", d), hp(iSp, d), hp(EWp, d)) if lp else (hp(P, d), hp("none", d), hp("none", d)))
    args_q = ((hp("none", m), hp(iSq, m), hp(EWq, m)) if lq else (hp(Q, m), hp("none", m), hp("none", m)))
    if P is not None and lp:
        args_p = (hp(P, d),) + args_p[1:]
    flags = L.PTR_DEVICE if flags is None else flags
    rc = ctx.lib.rxg_lgssm_vmp_noise_f32(
        ctx.h, d, m, T, nb, its, A.ctypes.data_as(L.fp), B.ctypes.data_as(L.fp), m0.ctypes.data_as(L.fp),
        S0.ctypes.data_as(L.fp), L.as_fp(0), args_p[0], nu_p, args_p[1], args_p[2], args_q[0], nu_q, args_q[1], args_q[2],
        p(y), ctypes.cast(c_void_p(None), L.u8p), p(mean), p(cov), op["df_p"], op["iS_p"], op["df_q"], op["iS_q"],
        ctypes.cast(c_void_p(None), ctypes.POINTER(ctypes.c_double)), ctypes.cast(c_void_p(None), L.i32p), flags)
    torch.cuda.synchronize()
    return rc


@pytest.mark.gpu
def test_refusals(ctx):
    from rxinfer_jl_b200 import _lib as L
    OK, U, BAD = L.RXG_OK, L.RXG_ERR_UNSUPPORTED, L.RXG_ERR_BAD_ARG
    assert _raw(ctx) == OK and _raw(ctx, learn="P") == OK and _raw(ctx, learn="Q") == OK
    assert _raw(ctx, flags=0, dev=False) == U                          # host data pointers
    for d, m in ((7, 2), (2, 7), (0, 2), (2, 0)):
        assert _raw(ctx, d=d, m=m) == U, (d, m)
    for f in (L.MODEL_PER_CHAIN, L.U_SEQ_SHARED, L.U_SEQ_CHAIN, L.COV_SHARED_OUT):
        assert _raw(ctx, flags=L.PTR_DEVICE | f) == U, f
    assert _raw(ctx, its=0) == BAD and _raw(ctx, T=0) == BAD
    assert _raw(ctx, learn="") == BAD                                   # both known: the plain smoother
    assert _raw(ctx, learn="PQ", P=np.eye(2)) == BAD                    # P and (inv_scale_p0, init_E_Wp) both given
    assert _raw(ctx, learn="P", EWp="none") == BAD and _raw(ctx, learn="P", iSp="none") == BAD   # half a pair
    assert _raw(ctx, learn="PQ", EWq="none") == BAD
    assert _raw(ctx, learn="P", outs=dict(df_p=False)) == BAD           # a learned noise needs its outputs
    assert _raw(ctx, learn="PQ", outs=dict(iS_q=False)) == BAD
    assert _raw(ctx, learn="P", outs=dict(df_q=True)) == BAD            # a known noise has none
    assert _raw(ctx, learn="Q", outs=dict(iS_p=True)) == BAD
    assert _raw(ctx, nu_p=1.0) == BAD and _raw(ctx, nu_p=0.5, d=1, m=1) == OK     # nu_p0 > d - 1
    assert _raw(ctx, nu_q=1.0) == BAD and _raw(ctx, learn="P", nu_q=0.0) == OK   # nu_q0 is ignored when Q is known
    assert _raw(ctx, nu_p=float("nan")) == BAD
    assert _raw(ctx, iSp=[[1.0, 2.0], [2.0, 1.0]]) == BAD               # not SPD
    assert _raw(ctx, EWp=[[1.0, 0.0], [0.0, -1.0]]) == BAD
    assert _raw(ctx, iSq=[[1.0, 2.0], [2.0, 1.0]]) == BAD
    assert _raw(ctx, EWq=[[0.0, 0.0], [0.0, 1.0]]) == BAD


@pytest.mark.gpu
def test_infer_pattern(ctx, rx):
    """infer(model = linear_gaussian_ssm_wishart_noise(...)) returns q(x) (KeepLast), q(w_p) and q(w_q) per iteration and
    the free energy; Wishart(df, scale) arguments are converted to the inverse scale and the mean."""
    from rxinfer_jl_b200 import inference as I
    from rxinfer_jl_b200.distributions import Wishart
    d, m, T, its = 3, 2, 30, 4
    mod, y, _, _ = random_problem(d, m, T, NB, seed=2)
    Sp, Sq = np.diag([4.0, 2.0, 1.0]), np.array([[1.5, 0.25], [0.25, 0.75]])
    model = I.linear_gaussian_ssm_wishart_noise(A=mod["A"], B=mod["B"], x0=(mod["m0"], mod["S0"]),
                                                p_prior=Wishart(5.0, Sp), p_init=Wishart(4.0, 2.0 * np.eye(d)),
                                                q_prior=Wishart(4.0, Sq), q_init=Wishart(3.0, 0.5 * np.eye(m)))
    res = I.infer(model=model, data={"y": torch.as_tensor(y, device="cuda")}, iterations=its, free_energy=True, context=ctx)
    ref = lgssm_wishart_noise(y, mod["A"], mod["B"], mod["m0"], mod["S0"], its, p_prior=(5.0, f32(np.linalg.inv(Sp))),
                              p_init=8.0 * np.eye(d), q_prior=(4.0, f32(np.linalg.inv(Sq))), q_init=1.5 * np.eye(m))
    wp, wq = res.posteriors["w_p"], res.posteriors["w_q"]
    assert tuple(wp.df.shape) == (its, NB) and tuple(wp.invS.shape) == (its, d, d, NB)
    assert tuple(wq.invS.shape) == (its, m, m, NB)
    assert res.free_energy.dtype == torch.float64 and tuple(res.free_energy.shape) == (its, NB)
    gate("infer", dict(mean=res.posteriors["x"].mu, cov=res.posteriors["x"].Sigma, df_p=wp.df, inv_scale_p=wp.invS,
                       df_q=wq.df, inv_scale_q=wq.invS, free_energy=res.free_energy), ref)
    model_p = I.linear_gaussian_ssm_wishart_noise(A=mod["A"], B=mod["B"], x0=(mod["m0"], mod["S0"]), Q=np.eye(m),
                                                  p_prior=Wishart(5.0, Sp), p_init=Wishart(4.0, 2.0 * np.eye(d)))
    res = I.infer(model=model_p, data={"y": torch.as_tensor(y, device="cuda")}, iterations=its, context=ctx)
    assert set(res.posteriors) == {"x", "w_p"}
