"""rxg_lgssm_vmp_wishart_f32 on the GPU: every chain gated against the fp64 reference of test_vmp_wishart.py at the
unchanged TOL_MEAN / TOL_COV (q(x), relative L2 / Frobenius per chain), TOL_COV for the inverse scale of q(w) at every
iteration (relative Frobenius per chain), df exactly and the free energy at TOL_NLE (relative to max(|F|, 1), per chain and
iteration); bit-exact relations with torch.equal; the cross-checks against the scalar Gamma kernel and the composed
per-chain path; the refusals of the C entry."""
import ctypes
from ctypes import c_void_p

import numpy as np
import pytest
import torch

from test_vmp_wishart import lgssm_wishart_precision, random_problem
from util import TOL_COV, TOL_MEAN, TOL_NLE

SHAPES = [(1, 1), (2, 1), (2, 2), (2, 3), (3, 3), (4, 2), (4, 4), (5, 3), (6, 6)]
NB = 7                                                   # odd batch


def _per_chain_rel(a, b, axes):
    a = np.asarray(a, np.float64); b = np.asarray(b, np.float64)
    num = np.sqrt(((a - b) ** 2).sum(axis=axes)); den = np.sqrt((b ** 2).sum(axis=axes))
    return num / np.maximum(den, 1e-30)


def gate(case, r, ref, its):
    mean, cov = r["mean"].cpu().numpy(), r["cov"].cpu().numpy()
    em = _per_chain_rel(mean, ref["mean"], (0, 1)); ec = _per_chain_rel(cov, ref["cov"], (0, 1, 2))
    assert em.max() <= TOL_MEAN, f"{case}: q(x) mean rel L2 {em.max():.3g} (chain {em.argmax()})"
    assert ec.max() <= TOL_COV, f"{case}: q(x) cov rel Frobenius {ec.max():.3g} (chain {ec.argmax()})"
    assert np.array_equal(r["df"].cpu().numpy().astype(np.float64), ref["df"]), f"{case}: df"
    ep = _per_chain_rel(r["inv_scale"].cpu().numpy(), ref["inv_scale"], (1, 2))        # [its, batch]
    assert ep.max() <= TOL_COV, f"{case}: inv_scale rel Frobenius {ep.max():.3g} at {np.unravel_index(ep.argmax(), ep.shape)}"
    if r["free_energy"] is not None:
        fe = r["free_energy"].cpu().numpy()
        ef = np.abs(fe - ref["free_energy"]) / np.maximum(np.abs(ref["free_energy"]), 1.0)
        assert ef.max() <= TOL_NLE, f"{case}: free energy rel {ef.max():.3g} at {np.unravel_index(ef.argmax(), ef.shape)}"


def monotone(fe, case):
    """F_k is non-increasing up to 2 TOL_NLE max(|F|, 1): the device values are within TOL_NLE of the fp64 sequence,
    which is non-increasing; smaller decreases are below the fp32 resolution of the terms."""
    fe = fe.double()
    slack = 2 * TOL_NLE * torch.clamp(fe[:-1].abs(), min=1.0)
    worst = (fe[1:] - fe[:-1] - slack).max().item() if fe.shape[0] > 1 else -1.0
    assert worst <= 0.0, f"{case}: free energy increased beyond the slack by {worst:.3g}"


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


def run(ctx, mod, y, its, *, mask=None, u=None, tf=False, W0=None, nu0=None, Psi0=None, fe=True):
    m = y.shape[1]
    nu0 = float(m + 2) if nu0 is None else nu0
    Psi0 = np.eye(m) * 0.5 if Psi0 is None else Psi0
    W0 = np.eye(m) if W0 is None else W0
    mk = None if mask is None else (torch.as_tensor(mask, device="cuda") if mask.ndim == 2 else mask)
    r = ctx.lgssm_vmp_wishart(torch.as_tensor(y, device="cuda"), mod["A"], mod["B"], mod["P"], mod["m0"], mod["S0"],
                              iterations=its, w_prior=(nu0, Psi0), init_E_W=W0, u=u, mask=mk, transition_first=tf,
                              want_free_energy=fe)
    torch.cuda.synchronize()
    return r, (nu0, Psi0, W0)


# (iterations, mask, transition_first, constant u, non-default init_E_W) per row: every (d, m, T) runs all three
VARIANTS = [(1, None, False, False, False), (5, "chain", True, True, False), (20, "shared", False, True, True)]


@pytest.mark.gpu
@pytest.mark.parametrize("T", [1, 2, 37, 300])
@pytest.mark.parametrize("d,m", SHAPES)
def test_matrix(ctx, d, m, T):
    mod, y, _, _ = random_problem(d, m, T, NB, seed=100 * d + 10 * m + T)
    for its, mk, tf, with_u, w0 in VARIANTS:
        case = f"d={d} m={m} T={T} its={its} mask={mk} tf={int(tf)} u={int(with_u)} W0={int(w0)}"
        u = np.linspace(-0.2, 0.3, d) if with_u else None
        W0 = (np.eye(m) * 3.0 + 0.4 * (np.ones((m, m)) - np.eye(m)) / m) if w0 else None
        mask = _mask(mk, T)
        r, (nu0, Psi0, W0) = run(ctx, mod, y, its, mask=mask, u=u, tf=tf, W0=W0)
        assert int(r["status"].abs().sum()) == 0, f"{case}: status {r['status'].tolist()}"
        ref = lgssm_wishart_precision(y, mod["A"], mod["B"], mod["P"], mod["m0"], mod["S0"], nu0, Psi0, W0, its,
                                      mask=mask, u=u, transition_first=tf)
        gate(case, r, ref, its)
        monotone(r["free_energy"], case)


@pytest.mark.gpu
@pytest.mark.parametrize("d,m", [(2, 2), (3, 3), (4, 4), (5, 3)])
def test_exact_relations(ctx, d, m):
    """A reversed batch gives the reversed results, a chain run alone equals the same chain inside the batch
    (torch.equal)."""
    T, its = 50, 6
    mod, y, _, _ = random_problem(d, m, T, NB, seed=5 * d + m)
    mask = _mask("chain", T)
    r, _ = run(ctx, mod, y, its, mask=mask)
    rr, _ = run(ctx, mod, np.ascontiguousarray(y[..., ::-1]), its, mask=np.ascontiguousarray(mask[:, ::-1]))
    for k in ("mean", "cov", "df", "inv_scale", "free_energy", "status"):
        assert torch.equal(rr[k].flip(-1), r[k]), k
    for c in (0, 3, NB - 1):
        r1, _ = run(ctx, mod, np.ascontiguousarray(y[..., c:c + 1]), its, mask=np.ascontiguousarray(mask[:, c:c + 1]))
        for k in ("mean", "cov", "df", "inv_scale", "free_energy"):
            assert torch.equal(r1[k][..., 0], r[k][..., c]), (k, c)


@pytest.mark.gpu
@pytest.mark.parametrize("d,m", [(2, 2), (3, 3), (4, 4), (4, 2)])
def test_one_iteration_is_the_per_chain_smoother(ctx, d, m):
    """iterations = 1 with init_E_W = inv(Q), Q diagonal with power-of-two entries (the fp64 inversion gives Q back
    exactly in fp32): q(x) equals Context.lgssm(..., force_per_chain_path=True), bit for bit -- both kernels run the
    same step helpers."""
    T = 40
    mod, y, _, _ = random_problem(d, m, T, NB, seed=9 * d + m)
    Q = np.diag([0.5, 2.0, 0.25, 1.0, 4.0, 0.125][:m])
    mask = _mask("chain", T)
    for tf, u, mk in ((False, None, None), (True, np.linspace(-0.1, 0.2, d), mask)):
        r, _ = run(ctx, mod, y, 1, mask=mk, u=u, tf=tf, W0=np.linalg.inv(Q), fe=False)
        yy = torch.as_tensor(y, device="cuda")
        ref = ctx.lgssm(yy, mod["A"], mod["B"], mod["P"], Q, mod["m0"], mod["S0"], u=u, smooth=True, force_per_chain_path=True,
                        mask=None if mk is None else torch.as_tensor(mk, device="cuda"), transition_first=tf)
        assert torch.equal(r["mean"], ref["mean"]) and torch.equal(r["cov"], ref["cov"]), (tf, mk is not None)


@pytest.mark.gpu
def test_scalar_case_matches_the_gamma_kernel(ctx):
    """d = m = 1 with nu0 = 2 a0, Psi0 = 2 b0 against rxg_lgssm_vmp_gamma_fe_f32 (a separate scalar fp32 implementation,
    so within tolerance, not bitwise)."""
    T, nb, its = 200, 33, 8
    rng = np.random.default_rng(17)
    y = (np.cumsum(rng.standard_normal((T, nb)), axis=0) + rng.standard_normal((T, nb)) * 0.6).astype(np.float32)
    a, v, (m0, v0), (a0, b0), Et = 0.95, 0.5, (0.0, 10.0), (1.5, 2.0), 0.8
    g = ctx.lgssm_vmp_gamma(torch.as_tensor(y, device="cuda"), iterations=its, a=a, v_proc=v, prior=(m0, v0),
                            gamma_prior=(a0, b0), init_E_tau=Et, want_free_energy=True)
    mod = dict(A=np.array([[a]]), B=np.eye(1), P=np.array([[v]]), m0=np.array([m0]), S0=np.array([[v0]]))
    r, _ = run(ctx, mod, y[:, None, :].copy(), its, W0=np.array([[Et]]), nu0=2 * a0, Psi0=np.array([[2 * b0]]))
    assert torch.equal(r["df"][-1], 2 * g["shape"])
    rel = lambda p, q: float((p.double() - q.double()).norm() / q.double().norm())
    assert rel(r["inv_scale"][-1, 0, 0], 2 * g["rate"]) < 1e-5
    assert rel(r["mean"][:, 0], g["mean"]) < 1e-5 and rel(r["cov"][:, 0, 0], g["var"]) < 1e-4
    assert rel(r["free_energy"], g["free_energy"]) < 1e-5


def composed_path(ctx, y, mod, its, nu0, Psi0, W0, mask=None, u=None):
    """What users compose today: per-chain Context.lgssm with Q_b = inv(E[w_b]), a torch reduction over T and the
    Wishart update in torch (fp64)."""
    T, m, nb = y.shape
    d = mod["A"].shape[0]
    dev = lambda M: torch.as_tensor(np.ascontiguousarray(np.broadcast_to(np.asarray(M, np.float32)[..., None],
                                                                          np.shape(M) + (nb,))), device="cuda")
    A, B, P, m0, S0 = (dev(mod[k]) for k in ("A", "B", "P", "m0", "S0"))
    uu = dev(u) if u is not None else None
    Bd = torch.as_tensor(mod["B"], dtype=torch.float64, device="cuda")
    Psi0t = torch.as_tensor(Psi0, dtype=torch.float64, device="cuda")
    W = torch.as_tensor(W0, dtype=torch.float64, device="cuda").unsqueeze(0).repeat(nb, 1, 1)
    mk = None if mask is None else torch.as_tensor(mask, device="cuda")
    obs = torch.ones(T, nb, dtype=torch.float64, device="cuda") if mk is None else mk.double()
    for _ in range(its):
        Q = torch.linalg.inv(W).permute(1, 2, 0).float().contiguous()
        r = ctx.lgssm(y, A, B, P, Q, m0, S0, u=uu, mask=mk, per_chain_model=True)
        e = y.double() - torch.einsum("kd,tdb->tkb", Bd, r["mean"].double())
        Rt = torch.einsum("tkb,tlb->tklb", e, e) + torch.einsum("kd,tdeb,le->tklb", Bd, r["cov"].double(), Bd)
        R = torch.einsum("tb,tklb->bkl", obs, Rt)
        df = nu0 + obs.sum(0)
        Psi = Psi0t + R
        W = df[:, None, None] * torch.linalg.inv(Psi)
    return dict(mean=r["mean"], cov=r["cov"], df=df, inv_scale=Psi.permute(1, 2, 0))


@pytest.mark.gpu
def test_fused_call_matches_the_composed_path(ctx):
    d, m, T, nb, its = 4, 4, 200, 256, 6
    mod, y_np, _, _ = random_problem(d, m, T, 8, seed=23)
    y_np = np.ascontiguousarray(np.tile(y_np, (1, 1, nb // 8)))
    y = torch.as_tensor(y_np, device="cuda")
    mask = np.ones((T, nb), dtype=np.uint8); mask[::7, ::3] = 0
    nu0, Psi0, W0 = 6.0, np.eye(m) * 0.5, np.eye(m)
    u = np.linspace(-0.2, 0.2, d)
    r = ctx.lgssm_vmp_wishart(y, mod["A"], mod["B"], mod["P"], mod["m0"], mod["S0"], iterations=its, w_prior=(nu0, Psi0),
                              init_E_W=W0, u=u, mask=torch.as_tensor(mask, device="cuda"))
    c = composed_path(ctx, y, mod, its, nu0, Psi0, W0, mask=mask, u=u)
    rel = lambda p, q: float((p.double() - q.double()).norm() / q.double().norm())
    assert torch.equal(r["df"][-1].double(), c["df"])
    assert rel(r["inv_scale"][-1], c["inv_scale"]) < TOL_COV
    assert rel(r["mean"], c["mean"]) < TOL_MEAN and rel(r["cov"], c["cov"]) < TOL_COV


@pytest.mark.gpu
def test_full_size(ctx):
    """d = m = 4, T = 1000, 65 536 chains, 10 iterations: every status OK, the free energy monotone for every chain, and
    64 sampled chains (both ends and the middle) against the reference."""
    d, m, T, nb, its = 4, 4, 1000, 65536, 10
    mod, y8, _, _ = random_problem(d, m, T, 64, seed=4)
    # 65 536 chains: the 64 seeded chains repeated with a per-chain perturbation of the data
    rng = np.random.default_rng(5)
    reps = nb // 64
    y = torch.as_tensor(y8, device="cuda").repeat(1, 1, reps)
    y += torch.as_tensor(rng.standard_normal((1, m, nb)).astype(np.float32) * 0.3, device="cuda")
    nu0, Psi0, W0 = 6.0, np.eye(m) * 0.5, np.eye(m)
    r = ctx.lgssm_vmp_wishart(y, mod["A"], mod["B"], mod["P"], mod["m0"], mod["S0"], iterations=its, w_prior=(nu0, Psi0),
                              init_E_W=W0, want_free_energy=True)
    torch.cuda.synchronize()
    assert int((r["status"] != 0).sum()) == 0
    monotone(r["free_energy"], "full size")
    idx = np.r_[0:22, nb // 2 - 10:nb // 2 + 10, nb - 22:nb]
    ys = y[..., idx].cpu().numpy()
    ref = lgssm_wishart_precision(ys, mod["A"], mod["B"], mod["P"], mod["m0"], mod["S0"], nu0, Psi0, W0, its)
    sub = {k: (v[..., idx] if v is not None else None) for k, v in r.items() if k != "status"}
    gate("full size", sub, ref, its)


# ====================================================================================== refusals
def _raw(ctx, d=2, m=2, T=4, nb=3, its=2, flags=None, nu0=4.0, iS0=None, W0=None, dev=True):
    from rxinfer_jl_b200 import _lib as L
    fp = lambda a: a.ctypes.data_as(L.fp)
    A = np.eye(d, dtype=np.float32); B = np.ones((m, d), np.float32); P = np.eye(d, dtype=np.float32)
    m0 = np.zeros(d, np.float32); S0 = np.eye(d, dtype=np.float32)
    iS0 = np.eye(m, dtype=np.float32) if iS0 is None else np.asarray(iS0, np.float32)
    W0 = np.eye(m, dtype=np.float32) if W0 is None else np.asarray(W0, np.float32)
    mm = max(m, 1); dd = max(d, 1)
    if dev:
        y = torch.zeros(T, mm, nb, device="cuda")
        mean, cov = torch.empty(T, dd, nb, device="cuda"), torch.empty(T, dd, dd, nb, device="cuda")
        df, iS = torch.empty(its if its > 0 else 1, nb, device="cuda"), torch.empty(max(its, 1), mm, mm, nb, device="cuda")
    else:
        y = torch.zeros(T, mm, nb)
        mean, cov = torch.empty(T, dd, nb), torch.empty(T, dd, dd, nb)
        df, iS = torch.empty(max(its, 1), nb), torch.empty(max(its, 1), mm, mm, nb)
    p = lambda t: L.as_fp(t.data_ptr())
    flags = L.PTR_DEVICE if flags is None else flags
    rc = ctx.lib.rxg_lgssm_vmp_wishart_f32(ctx.h, d, m, T, nb, its, fp(A), fp(B), fp(P), fp(m0), fp(S0), L.as_fp(0), nu0,
                                           fp(iS0), fp(W0), p(y), ctypes.cast(c_void_p(None), L.u8p), p(mean), p(cov), p(df),
                                           p(iS), ctypes.cast(c_void_p(None), ctypes.POINTER(ctypes.c_double)),
                                           ctypes.cast(c_void_p(None), L.i32p), flags)
    torch.cuda.synchronize()
    return rc


@pytest.mark.gpu
def test_refusals(ctx):
    from rxinfer_jl_b200 import _lib as L
    assert _raw(ctx) == L.RXG_OK
    U, BAD = L.RXG_ERR_UNSUPPORTED, L.RXG_ERR_BAD_ARG
    assert _raw(ctx, flags=0, dev=False) == U                         # host data pointers
    for d, m in ((7, 2), (2, 7), (0, 2), (2, 0)):
        assert _raw(ctx, d=d, m=m) == U, (d, m)
    for f in (L.MODEL_PER_CHAIN, L.U_SEQ_SHARED, L.U_SEQ_CHAIN, L.COV_SHARED_OUT):
        assert _raw(ctx, flags=L.PTR_DEVICE | f) == U, f
    assert _raw(ctx, its=0) == BAD
    assert _raw(ctx, nu0=1.0) == BAD and _raw(ctx, nu0=0.5, m=1, d=1) == L.RXG_OK    # nu0 > m - 1
    assert _raw(ctx, iS0=[[1.0, 2.0], [2.0, 1.0]]) == BAD              # not SPD
    assert _raw(ctx, W0=[[1.0, 0.0], [0.0, -1.0]]) == BAD


@pytest.mark.gpu
def test_infer_pattern(ctx, rx):
    """infer(model = linear_gaussian_ssm_wishart_precision(...)) returns q(x) (KeepLast), q(w) per iteration and the
    free energy; the Wishart(df, scale) arguments are converted to the inverse scale and the mean."""
    from rxinfer_jl_b200 import inference as I
    from rxinfer_jl_b200.distributions import Wishart
    d, m, T, its = 3, 2, 30, 4
    mod, y, _, _ = random_problem(d, m, T, NB, seed=2)
    S = np.array([[1.5, 0.2], [0.2, 0.8]])
    model = I.linear_gaussian_ssm_wishart_precision(A=mod["A"], B=mod["B"], P=mod["P"], x0=(mod["m0"], mod["S0"]),
                                                    w_prior=Wishart(4.0, S), w_init=Wishart(3.0, 0.5 * np.eye(m)))
    res = I.infer(model=model, data={"y": torch.as_tensor(y, device="cuda")}, iterations=its, free_energy=True, context=ctx)
    ref = lgssm_wishart_precision(y, mod["A"], mod["B"], mod["P"], mod["m0"], mod["S0"], 4.0, np.linalg.inv(S), 1.5 * np.eye(m), its)
    w = res.posteriors["w"]
    assert tuple(w.df.shape) == (its, NB) and tuple(w.invS.shape) == (its, m, m, NB)
    assert res.free_energy.dtype == torch.float64 and tuple(res.free_energy.shape) == (its, NB)
    gate("infer", dict(mean=res.posteriors["x"].mu, cov=res.posteriors["x"].Sigma, df=w.df, inv_scale=w.invS,
                       free_energy=res.free_energy), ref, its)
