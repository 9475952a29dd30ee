"""rxg_hmm_gauss_vmp_f32 on the GPU: every chain gated against the fp64 reference of test_hmm_gauss.py, which gets the
fp32-rounded inputs.  Per chain: E[m], alpha_A, nu at TOL_MEAN relative L2; cov m and the W inverse scale at TOL_COV;
q(s_t), q(s_0) at 10 TOL_COV absolute; the KeepEach histories at 3x those; the free energy at FE_TOL relative to
max(|F|, 1) at the last iteration, 2 FE_TOL at the earlier ones, and non-increasing.  Then long series, half the steps missing, far-from-origin clusters, a sticky
A, flagged chains beside healthy ones, bit-exact batch reversal and slices, the KeepEach final slots against the
last-iteration outputs, the C entry's refusals, and infer in both spellings with the recovery assertions."""
import numpy as np
import pytest
import torch

from test_hmm_gauss import gate, random_problem, recovery_assertions, recovery_problem, reference_on_f32
from util import TOL_COV, TOL_MEAN

pytestmark = pytest.mark.gpu
NB = 7                                         # odd batch
FE_TOL = 1e-5


def run(ctx, y, kw, its, **extra):
    r = ctx.hmm_gauss_vmp(torch.as_tensor(np.asarray(y, np.float32), device="cuda:0").contiguous(),
                          **{k: np.asarray(v, np.float32) for k, v in kw.items()}, iterations=its, keep_each=True, **extra)
    return {k: (v.cpu().numpy() if v is not None else None) for k, v in r.items()}


def check(case, r, y, kw, its, chains=None):
    """The gates of the module docstring.  F: FE_TOL at the last iteration; 2 FE_TOL at the earlier ones, where a chain
    whose iteration crosses an ill-conditioned stretch departs from the fp64 trajectory for a few iterations before it
    reconverges (DESIGN 3.20)."""
    ref = reference_on_f32(y, kw, its)
    w = gate(case, r, ref, chains=chains, tol_mean=TOL_MEAN, tol_cov=TOL_COV, tol_s=10 * TOL_COV, fe_tol=2 * FE_TOL)
    sel = (lambda v: v[..., chains]) if chains is not None else (lambda v: v)
    fe, fr = sel(np.asarray(r["free_energy"]))[-1], sel(ref["free_energy"])[-1]
    e = (np.abs(fe - fr) / np.maximum(np.abs(fr), 1.0)).max()
    assert e < FE_TOL, f"{case}: last-iteration free energy {e:.3g}"
    w["free_energy_last"] = e
    return w


def _worst(acc, w):
    for k, v in w.items():
        acc[k] = max(acc.get(k, 0.0), float(v))


@pytest.mark.parametrize("K", [2, 3, 5, 8])
@pytest.mark.parametrize("d", [1, 2, 3, 4])
def test_every_chain_against_the_fp64_reference(ctx, d, K):
    worst = {}
    for T in (1, 7, 1000):
        for la in (True, False):
            y, kw = random_problem(d, K, T, NB, seed=1000 * d + 10 * K + T + la, learn_A=la, p_missing=0.1)
            for its in (1, 20):
                _worst(worst, check(f"d={d} K={K} T={T} its={its} learn A={la}", run(ctx, y, kw, its), y, kw, its))
    print(f"worst d={d} K={K}", {k: f"{v:.3g}" for k, v in sorted(worst.items())})


def test_long_series_half_missing_far_clusters_and_a_sticky_a(ctx):
    y, kw = random_problem(2, 4, 10000, 3, seed=11)
    check("T=10000", run(ctx, y, kw, 5), y, kw, 5)
    y, kw = random_problem(3, 5, 400, NB, seed=12, p_missing=0.5)
    check("half missing", run(ctx, y, kw, 10), y, kw, 10)
    for d, K in ((1, 2), (2, 3), (4, 8)):     # 100 from the origin, as far as the mixture's test (DESIGN 3.20)
        y, kw = random_problem(d, K, 300, NB, seed=13 + d, offset=100.0)
        check(f"far clusters d={d} K={K}", run(ctx, y, kw, 10), y, kw, 10)
    for la in (True, False):
        y, kw = random_problem(2, 3, 500, NB, seed=14, learn_A=la, sharp=True)
        if la:
            kw["A_prior"] = kw["A_prior"] + 50.0 * np.eye(3)
        check(f"sticky A learned={la}", run(ctx, y, kw, 8), y, kw, 8)


def test_flagged_chains_leave_their_neighbours_alone(ctx):
    y, kw = random_problem(2, 3, 60, NB, seed=15, p_missing=0.1)
    y[5, 0, 1] = np.inf                                       # a non-finite datum: BAD_ARG, the step read as missing
    y[8, 1, 3] = np.nan                                       # one component NaN only: BAD_ARG as well
    y[3, :, 5] = 3e38                                         # every emission weight vanishes: NAN
    r = run(ctx, y, kw, 4)
    assert list(r["status"]) == [0, 1, 0, 1, 0, 5, 0]
    ym = y.copy()
    ym[:, :, [1, 3, 5]] = np.nan                             # the reference of the healthy chains only
    check("flagged neighbours", r, ym, kw, 4, chains=[0, 2, 4, 6])


def test_batch_reversal_and_slices_are_bit_exact(ctx):
    y, kw = random_problem(3, 4, 200, 9, seed=16, p_missing=0.1)
    r = run(ctx, y, kw, 6)
    rr = run(ctx, y[..., ::-1].copy(), kw, 6)
    rs = run(ctx, y[..., 2:7].copy(), kw, 6)
    for k, v in r.items():
        if v is None:
            continue
        assert np.array_equal(rr[k], v[..., ::-1]), k
        assert np.array_equal(rs[k], v[..., 2:7]), k


def test_keep_each_final_slot_equals_the_last_iteration_bit_for_bit(ctx):
    y, kw = random_problem(2, 6, 120, NB, seed=17, p_missing=0.2)
    yd = torch.as_tensor(np.asarray(y, np.float32), device="cuda:0")
    k32 = {k: np.asarray(v, np.float32) for k, v in kw.items()}
    r = ctx.hmm_gauss_vmp(yd, **k32, iterations=7, keep_each=True)
    for k in ("s", "A", "m_mean", "m_cov", "w_df", "w_inv_scale"):
        last = r["s_prob"] if k == "s" else r["A_alpha"] if k == "A" else r[k]
        assert torch.equal(r["hist_" + k][-1], last), k
    r1 = ctx.hmm_gauss_vmp(yd, **k32, iterations=7, want_free_energy=False)
    assert r1["free_energy"] is None and "hist_s" not in r1
    for k in ("s_prob", "s0_prob", "A_alpha", "m_mean", "w_inv_scale"):
        assert torch.equal(r1[k], r[k]), k


def test_c_entry_refusals(ctx, rx):
    y, kw = random_problem(2, 3, 10, 2, seed=18)
    yd = torch.as_tensor(np.asarray(y, np.float32), device="cuda:0")
    k32 = {k: np.asarray(v, np.float32) for k, v in kw.items()}
    indefinite = np.array([[1.0, 2.0], [2.0, 1.0]], np.float32)
    bad_cases = [dict(k32, A_known=np.eye(3, dtype=np.float32)),                          # both A choices
                 {k: v for k, v in k32.items() if k != "A_init"},                          # prior without init
                 {k: v for k, v in k32.items() if k not in ("A_prior", "A_init")},         # neither
                 dict(k32, A_prior=-k32["A_prior"]),                                       # Dirichlet parameter <= 0
                 dict(k32, p0=np.array([0.5, 0.5, 0.5], np.float32)),                      # p0 sums to 1.5
                 dict({k: v for k, v in k32.items() if not k.startswith("A_")},
                      A_known=np.full((3, 3), 0.4, np.float32)),                           # columns sum to 1.2
                 dict(k32, nu0=np.full(3, 0.9, np.float32)),                               # nu <= d - 1
                 dict(k32, nu_init=np.full(3, 1.0, np.float32))]
    for name in ("V0", "S0", "Vm_init", "S_init"):                                         # not SPD
        a = k32[name].copy()
        a[1] = indefinite
        bad_cases.append(dict(k32, **{name: a}))
    for c in bad_cases:
        with pytest.raises(rx.RxGaussError) as e:
            ctx.hmm_gauss_vmp(yd, **c)
        assert e.value.code == rx._lib.RXG_ERR_BAD_ARG, [k for k in c if c[k] is not k32.get(k)]
    for d, K in ((5, 3), (2, 9), (2, 1)):                                                   # d or K out of range
        yd5 = torch.zeros(5, d, 2, device="cuda:0")
        k5 = dict(p0=np.full(K, 1 / K, np.float32), A_prior=np.ones((K, K), np.float32), A_init=np.ones((K, K), np.float32),
                  mu0=np.zeros((K, d), np.float32), V0=np.tile(np.eye(d, dtype=np.float32), (K, 1, 1)),
                  nu0=np.full(K, d + 1.0, np.float32), S0=np.tile(np.eye(d, dtype=np.float32), (K, 1, 1)),
                  m_init=np.zeros((K, d), np.float32), Vm_init=np.tile(np.eye(d, dtype=np.float32), (K, 1, 1)),
                  nu_init=np.full(K, d + 1.0, np.float32), S_init=np.tile(np.eye(d, dtype=np.float32), (K, 1, 1)))
        with pytest.raises(rx.RxGaussError) as e:
            ctx.hmm_gauss_vmp(yd5, **k5)
        assert e.value.code == rx._lib.RXG_ERR_UNSUPPORTED, (d, K)
    # sizes below 1, and host pointers
    keep = {k: np.ascontiguousarray(v) for k, v in k32.items()}
    P = lambda a: a.ctypes.data_as(rx._lib.fp)
    A = [P(keep[k]) for k in ("p0", "A_prior", "A_init")] + [None] + [P(keep[k]) for k in
                                                                       ("mu0", "V0", "nu0", "S0", "m_init", "Vm_init",
                                                                        "nu_init", "S_init")]
    out = torch.empty(10, 3, 2, device="cuda:0")
    yp = rx._lib.as_fp(yd.data_ptr())
    op = rx._lib.as_fp(out.data_ptr())
    for T, nb, its in ((0, 2, 1), (10, 0, 1), (10, 2, 0)):
        rc = ctx.lib.rxg_hmm_gauss_vmp_f32(ctx.h, 2, 3, T, nb, its, *A, yp, op, *([None] * 14), rx._lib.PTR_DEVICE)
        assert rc == rx._lib.RXG_ERR_BAD_ARG, (T, nb, its)
    rc = ctx.lib.rxg_hmm_gauss_vmp_f32(ctx.h, 2, 3, 10, 2, 1, *A, yp, op, *([None] * 14), 0)
    assert rc == rx._lib.RXG_ERR_UNSUPPORTED


def test_infer_in_both_spellings_and_recovery_on_the_cuda_output(ctx, rx):
    from rxinfer_jl_b200 import (DirichletCollection, GammaShapeRate, GaussianHMMConstraints, KeepEach,
                                 MvNormalMeanCovariance, NormalMeanVariance, Wishart, gaussian_hidden_markov_model)
    y, s_true, means, A, kw = recovery_problem(nb=NB)
    model = gaussian_hidden_markov_model(p0=kw["p0"], A=DirichletCollection(kw["A_prior"]),
                                         m_prior=[MvNormalMeanCovariance(kw["mu0"][k], kw["V0"][k]) for k in range(3)],
                                         w_prior=[Wishart(kw["nu0"][k], kw["S0"][k]) for k in range(3)])
    init = {"A": DirichletCollection(kw["A_init"]), "m": [MvNormalMeanCovariance(kw["m_init"][k], kw["Vm_init"][k])
                                                           for k in range(3)],
            "w": [Wishart(kw["nu_init"][k], kw["S_init"][k]) for k in range(3)]}
    res = rx.infer(model=model, constraints=GaussianHMMConstraints(), data={"y": torch.as_tensor(y, dtype=torch.float32)},
                   initialization=init, iterations=30, free_energy=True, returnvars={"s": KeepEach(), "m": KeepEach()},
                   context=ctx)
    assert res.posteriors["s"].p.shape == (30, 1000, 3, NB) and res.posteriors["A"].alpha.shape == (3, 3, NB)
    r = dict(m_mean=torch.stack([res.posteriors["m"][k].mu[-1] for k in range(3)]).cpu().numpy(),
             A_alpha=res.posteriors["A"].alpha.cpu().numpy(), s_prob=res.posteriors["s"].p[-1].cpu().numpy())
    for b in range(NB):
        recovery_assertions(r, s_true, means, A, b=b)
    ref = reference_on_f32(y, kw, 30)
    fe = res.free_energy.cpu().numpy()
    assert (np.abs(fe - ref["free_energy"]) / np.maximum(np.abs(ref["free_energy"]), 1.0)).max() < FE_TOL
    # the univariate spelling at d = 1: NormalMeanVariance / GammaShapeRate, data as [T, batch]
    y1, kw1 = random_problem(1, 2, 200, NB, seed=20)
    m1 = gaussian_hidden_markov_model(p0=kw1["p0"], A=DirichletCollection(kw1["A_prior"]),
                                      m_prior=[NormalMeanVariance(kw1["mu0"][k, 0], kw1["V0"][k, 0, 0]) for k in range(2)],
                                      w_prior=[GammaShapeRate(kw1["nu0"][k] / 2, 1 / (2 * kw1["S0"][k, 0, 0]))
                                               for k in range(2)])
    i1 = {"A": DirichletCollection(kw1["A_init"]),
          "m": [NormalMeanVariance(kw1["m_init"][k, 0], kw1["Vm_init"][k, 0, 0]) for k in range(2)],
          "w": [GammaShapeRate(kw1["nu_init"][k] / 2, 1 / (2 * kw1["S_init"][k, 0, 0])) for k in range(2)]}
    res1 = rx.infer(model=m1, constraints=GaussianHMMConstraints(), data={"y": torch.as_tensor(y1[:, 0], dtype=torch.float32)},
                    initialization=i1, iterations=10, free_energy=True, context=ctx)
    ref1 = reference_on_f32(y1, kw1, 10)
    for k in range(2):
        q = res1.posteriors["m"][k]
        assert np.abs(q.m.cpu().numpy() - ref1["m_mean"][k, 0]).max() < 1e-4 * max(1.0, np.abs(ref1["m_mean"]).max())
        w = res1.posteriors["w"][k]
        assert np.abs(2 * w.a.cpu().numpy() - ref1["w_df"][k]).max() < 1e-4 * np.abs(ref1["w_df"]).max()
    fe1 = res1.free_energy.cpu().numpy()
    assert (np.abs(fe1 - ref1["free_energy"]) / np.maximum(np.abs(ref1["free_energy"]), 1.0)).max() < FE_TOL
    # flagged chains raise, as the HMM does
    bad = torch.as_tensor(y, dtype=torch.float32).clone()
    bad[4, 0, 1] = float("inf")
    with pytest.raises(rx.RxGaussError, match="1 of 7 chains"):
        rx.infer(model=model, constraints=GaussianHMMConstraints(), data={"y": bad}, initialization=init, iterations=2,
                 context=ctx)
