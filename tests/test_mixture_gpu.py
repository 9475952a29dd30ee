"""rxg_gmm_vmp_f32 on the GPU: every chain gated against the fp64 reference of test_mixture.py, which gets the
fp32-rounded inputs.  Per chain: the q(m) means and q(s) / q(W) degrees of freedom at TOL_MEAN, the q(m) covariances and
q(W) inverse scales at TOL_COV (relative L2 / Frobenius over all components and, for the histories, all iterations), q(z)
at 10 TOL_COV absolute, the free energy at FE_TOL relative to max(|F|, 1) per chain and iteration.  The KeepEach
histories of q(m) and q(W) are gated at 3 TOL_MEAN / 3 TOL_COV: the early iterates of a slowly converging chain amplify the
fp32 rounding of the responsibilities (measured worst 1.2e-4 on a q(m) covariance history, DESIGN 3.17).  Bit-exact
relations with torch.equal; the reference tests' assertions on the CUDA output; every refusal of the C entry; infer."""
import ctypes
from ctypes import c_void_p

import numpy as np
import pytest
import torch

from test_mixture import (PRIOR_KEYS, f32, gaussian_mixture, multivariate_assertions, multivariate_reference_data,
                          multivariate_reference_model, problem, univariate_assertions, univariate_reference_data,
                          univariate_reference_model)
from util import TOL_COV, TOL_MEAN

pytestmark = pytest.mark.gpu
NB = 7                                         # odd batch
FE_TOL = 1e-5
GATES = dict(alpha=TOL_MEAN, w_df=TOL_MEAN, m_mean=TOL_MEAN, m_cov=TOL_COV, w_inv_scale=TOL_COV,
             hist_alpha=3 * TOL_MEAN, hist_w_df=3 * TOL_MEAN, hist_m_mean=3 * TOL_MEAN, hist_m_cov=3 * TOL_COV,
             hist_w_inv_scale=3 * TOL_COV)


def dev(a):
    return torch.as_tensor(np.asarray(a, np.float32), device="cuda:0").contiguous()


def run(ctx, y, pri, its, **kw):
    """CUDA and fp64 reference on the same fp32-rounded inputs."""
    y32 = f32(y)
    p32 = {k: f32(v) for k, v in pri.items()}
    r = ctx.gmm_vmp(dev(y32), *(p32[k] for k in PRIOR_KEYS), iterations=its, want_z=True, keep_each=True, **kw)
    ref = gaussian_mixture(y32, **p32, iterations=its)
    return r, ref


def gate(case, r, ref):
    assert int(r["status"].abs().sum()) == 0, case
    for k, tol in GATES.items():
        got = r[k].cpu().numpy().astype(np.float64)
        want = ref[k]
        ax = tuple(range(got.ndim - 1))
        err = np.sqrt(((got - want) ** 2).sum(ax)) / np.maximum(np.sqrt((want ** 2).sum(ax)), 1e-30)
        assert err.max() < tol, f"{case}: {k} worst chain {int(err.argmax())} err {err.max():.3g} > {tol}"
    ez = np.abs(r["z_prob"].cpu().numpy() - ref["z_prob"]).max()
    assert ez < 10 * TOL_COV, f"{case}: z_prob {ez:.3g}"
    fe = r["free_energy"].cpu().numpy()
    efe = np.abs(fe - ref["free_energy"]) / np.maximum(np.abs(ref["free_energy"]), 1.0)
    assert efe.max() < FE_TOL, f"{case}: free energy {efe.max():.3g}"
    return fe


@pytest.mark.parametrize("K", [2, 3, 5, 8])
@pytest.mark.parametrize("d", [1, 2, 3, 4])
def test_every_chain_against_the_fp64_reference(ctx, d, K):
    for N in (1, 7, 500):
        for its in (1, 25):
            overlap = (N + its) % 2 == 0                 # separated and overlapping clusters
            y, pri = problem(d, K, N, NB, seed=1000 * d + 100 * K + N + its, overlap=overlap)
            r, ref = run(ctx, y, pri, its)
            fe = gate(f"d={d} K={K} N={N} its={its} overlap={overlap}", r, ref)
            slack = 2 * FE_TOL * np.maximum(np.abs(fe[:-1]), 1.0)
            assert np.all(np.diff(fe, axis=0) <= slack), (d, K, N, its)


@pytest.mark.parametrize("d,K", [(1, 2), (2, 3), (4, 8)])
def test_far_from_origin_clusters_meet_the_same_gates(ctx, d, K):
    """Clusters at radius 50 around a centre 50 away from the origin, as in the reference's multivariate test: the
    statistics are accumulated around the previous E[m_k] in fp64."""
    y, pri = problem(d, K, 500, NB, seed=77 + d, radius=50.0)
    shift = np.full(d, 50.0)
    y = y + shift[None, :, None]
    pri = dict(pri, mu0=pri["mu0"] + shift, m_init=pri["m_init"] + shift)
    r, ref = run(ctx, y, pri, 25)
    gate(f"far d={d} K={K}", r, ref)


def test_batch_reversal_and_slices_are_bit_exact(ctx):
    y, pri = problem(3, 5, 300, 9, seed=5)
    args = [f32(pri[k]) for k in PRIOR_KEYS]
    yd = dev(y)
    full = ctx.gmm_vmp(yd, *args, iterations=12, want_z=True, keep_each=True)
    rev = ctx.gmm_vmp(yd.flip(-1).contiguous(), *args, iterations=12, want_z=True, keep_each=True)
    part = ctx.gmm_vmp(yd[..., 3:5].contiguous(), *args, iterations=12, want_z=True, keep_each=True)
    for k, v in full.items():
        assert torch.equal(rev[k].flip(-1), v), k
        assert torch.equal(part[k], v[..., 3:5]), k
    lean = ctx.gmm_vmp(yd, *args, iterations=12, want_free_energy=False)          # optional outputs change nothing
    for k in ("alpha", "m_mean", "m_cov", "w_df", "w_inv_scale", "status"):
        assert torch.equal(lean[k], full[k]), k
    assert torch.equal(full["hist_m_mean"][-1], full["m_mean"]) and torch.equal(full["hist_w_inv_scale"][-1], full["w_inv_scale"])


def _np(r):
    return {k: (v.cpu().numpy().astype(np.float64) if v is not None else None) for k, v in r.items()}


def test_reference_assertions_on_the_cuda_output(ctx):
    y, switch, mus, ws = univariate_reference_data()
    _, _, arr = univariate_reference_model()
    r = ctx.gmm_vmp(dev(y[:, None, None]), *(arr[k] for k in PRIOR_KEYS), iterations=10, keep_each=True)
    univariate_assertions(_np(r), switch, mus, ws)
    y, means = multivariate_reference_data()
    _, _, arr = multivariate_reference_model()
    r = ctx.gmm_vmp(dev(y[:, :, None]), *(arr[k] for k in PRIOR_KEYS), iterations=25, keep_each=True)
    multivariate_assertions(_np(r), means)


def test_a_chain_with_a_non_finite_datum_is_flagged_and_the_others_are_not_touched(ctx):
    y, pri = problem(2, 3, 50, NB, seed=8)
    args = [f32(pri[k]) for k in PRIOR_KEYS]
    good = ctx.gmm_vmp(dev(y), *args, iterations=5)
    y[10, 1, 4] = np.nan
    bad = ctx.gmm_vmp(dev(y), *args, iterations=5)
    from rxinfer_jl_b200 import _lib as L
    assert bad["status"].tolist() == [0, 0, 0, 0, L.RXG_ERR_NOT_SPD, 0, 0]
    keep = [0, 1, 2, 3, 5, 6]
    for k in ("alpha", "m_mean", "m_cov", "w_df", "w_inv_scale", "free_energy"):
        assert torch.equal(bad[k][..., keep], good[k][..., keep]), k


def _code(fn, *a, **k):
    from rxinfer_jl_b200 import _lib as L
    with pytest.raises(L.RxGaussError) as e:
        fn(*a, **k)
    return e.value.code


def test_refusals(ctx):
    from rxinfer_jl_b200 import _lib as L
    U, BAD = L.RXG_ERR_UNSUPPORTED, L.RXG_ERR_BAD_ARG

    def args(d, K, **over):
        a = dict(alpha0=np.ones(K), mu0=np.zeros((K, d)), V0=np.tile(np.eye(d), (K, 1, 1)), nu0=np.full(K, d + 1.0),
                 S0=np.tile(np.eye(d), (K, 1, 1)), alpha_init=np.ones(K), m_init=np.zeros((K, d)),
                 Vm_init=np.tile(np.eye(d), (K, 1, 1)), nu_init=np.full(K, d + 1.0), S_init=np.tile(np.eye(d), (K, 1, 1)))
        a.update(over)
        return [a[k] for k in PRIOR_KEYS]

    y2 = dev(np.ones((4, 2, 3)))
    assert int(ctx.gmm_vmp(y2, *args(2, 3))["status"].abs().sum()) == 0
    # shapes outside d 1..4, K 2..8
    assert _code(ctx.gmm_vmp, dev(np.ones((4, 5, 3))), *args(5, 3)) == U
    assert _code(ctx.gmm_vmp, y2, *args(2, 1)) == U
    assert _code(ctx.gmm_vmp, y2, *args(2, 9)) == U
    # sizes
    assert _code(ctx.gmm_vmp, dev(np.ones((0, 2, 3))), *args(2, 3)) == BAD
    assert _code(ctx.gmm_vmp, y2, *args(2, 3), iterations=0) == BAD
    # hyper-parameters
    bad_spd = np.tile(np.array([[1.0, 2.0], [2.0, 1.0]]), (3, 1, 1))
    for over in (dict(alpha0=np.array([1.0, 0.0, 1.0])), dict(alpha_init=np.array([1.0, -1.0, 1.0])),
                 dict(nu0=np.array([3.0, 1.0, 3.0])), dict(nu_init=np.array([3.0, 3.0, 0.5])),
                 dict(V0=bad_spd), dict(S0=bad_spd), dict(Vm_init=bad_spd), dict(S_init=bad_spd),
                 dict(mu0=np.full((3, 2), np.nan)), dict(m_init=np.full((3, 2), np.inf)),
                 dict(alpha0=np.array([1.0, np.nan, 1.0]))):
        assert _code(ctx.gmm_vmp, y2, *args(2, 3, **over)) == BAD, over
    assert int(ctx.gmm_vmp(y2, *args(2, 3, nu0=np.full(3, 1.01), nu_init=np.full(3, 1.5)))["status"].abs().sum()) == 0
    # matrices built as R D R' are asymmetric in the last bit; the symmetrised part is what is checked and used
    a = 0.7
    R = np.array([[np.cos(a), -np.sin(a)], [np.sin(a), np.cos(a)]])
    C = (R @ np.diag([10.0, 20.0]) @ R.T).astype(np.float32)
    C[0, 1] = np.nextafter(C[1, 0], np.float32(np.inf))
    assert C[0, 1] != C[1, 0]
    Cs = np.tile(C.astype(np.float64), (3, 1, 1))
    r_asym = ctx.gmm_vmp(y2, *args(2, 3, V0=Cs, S0=Cs, Vm_init=Cs, S_init=Cs))
    Csym = np.tile(0.5 * (C.astype(np.float64) + C.T.astype(np.float64)), (3, 1, 1))
    r_sym = ctx.gmm_vmp(y2, *args(2, 3, V0=Csym, S0=Csym, Vm_init=Csym, S_init=Csym))
    assert int(r_asym["status"].abs().sum()) == 0
    assert torch.allclose(r_asym["m_cov"], r_sym["m_cov"], rtol=1e-6) and torch.allclose(r_asym["m_mean"], r_sym["m_mean"], rtol=1e-6)
    # the host-side shape checks of Context
    with pytest.raises(ValueError):
        ctx.gmm_vmp(y2, *args(3, 3))
    # host pointers and null required pointers in the C entry
    lib = ctx.lib
    fpn = ctypes.cast(c_void_p(None), L.fp)
    hp = [np.ascontiguousarray(np.asarray(a, np.float32)) for a in args(2, 3)]
    hpp = [a.ctypes.data_as(L.fp) for a in hp]
    outs = [torch.empty(n, device="cuda:0") for n in (9, 18, 36, 9, 36)]
    op = [ctypes.cast(c_void_p(t.data_ptr()), L.fp) for t in outs]
    dn = ctypes.cast(c_void_p(None), ctypes.POINTER(ctypes.c_double))
    i32n = ctypes.cast(c_void_p(None), L.i32p)
    yp = ctypes.cast(c_void_p(y2.data_ptr()), L.fp)
    call = lambda y_, o0, flags: lib.rxg_gmm_vmp_f32(ctx.h, 2, 3, 4, 3, 2, *hpp, y_, o0, *op[1:], dn, fpn, fpn, fpn, fpn, fpn,
                                                      fpn, i32n, flags)
    assert call(yp, op[0], L.PTR_DEVICE) == L.RXG_OK
    assert call(yp, op[0], 0) == U
    assert call(fpn, op[0], L.PTR_DEVICE) == BAD
    assert call(yp, fpn, L.PTR_DEVICE) == BAD
    assert lib.rxg_gmm_vmp_f32(None, 2, 3, 4, 3, 2, *hpp, yp, *op, dn, fpn, fpn, fpn, fpn, fpn, fpn, i32n,
                               L.PTR_DEVICE) == BAD


def test_infer_end_to_end(ctx, rx):
    from rxinfer_jl_b200.inference import BetheFactorization, MeanField
    y, means = multivariate_reference_data(n=200)
    ys = np.stack([y, y[::-1] + 1.0, y * 0.9], axis=-1)                  # three data sets [N, 2, 3]
    model, init, arr = multivariate_reference_model()
    res = rx.infer(model=model, data={"y": dev(ys)}, initialization=init, iterations=25, returnvars=rx.KeepEach(),
                   free_energy=True, constraints=MeanField(), context=ctx)
    ref = gaussian_mixture(f32(ys), **{k: f32(arr[k]) for k in PRIOR_KEYS}, iterations=25)
    assert res.posteriors["s"].alpha.shape == (25, 3, 3)
    assert len(res.posteriors["m"]) == 3 and res.posteriors["m"][0].mu.shape == (25, 2, 3)
    got = torch.stack([q.mu for q in res.posteriors["m"]], dim=1).cpu().numpy()          # [25, K, d, B]
    assert np.abs(got - ref["hist_m_mean"]).max() < 1e-3
    assert np.abs(res.free_energy.cpu().numpy() - ref["free_energy"]).max() < FE_TOL * np.abs(ref["free_energy"]).max()
    assert res.posteriors["z"].p.shape == (200, 3, 3)
    last = rx.infer(model=model, data={"y": dev(ys)}, initialization=init, iterations=25, returnvars=rx.KeepLast(),
                    constraints=MeanField(), context=ctx)
    assert torch.equal(last.posteriors["w"][1].invS, res.posteriors["w"][1].invS[-1])
    with pytest.raises(ValueError, match="must be the naive mean-field"):
        rx.infer(model=model, data={"y": dev(ys)}, initialization=init, iterations=2, constraints=BetheFactorization(),
                 context=ctx)
    with pytest.raises(ValueError, match="must be the naive mean-field"):
        rx.infer(model=model, data={"y": dev(ys)}, initialization=init, iterations=2, context=ctx)
    # the univariate spelling: Beta / Normal / Gamma posteriors
    yu, switch, mus, ws = univariate_reference_data()
    umodel, uinit, _ = univariate_reference_model()
    ru = rx.infer(model=umodel, data={"y": dev(yu[:, None])}, initialization=uinit, iterations=10, returnvars=rx.KeepEach(),
                  free_energy=True, constraints=MeanField(), context=ctx)
    s = ru.posteriors["s"]
    assert s.a.shape == (10, 1)
    ms = float((s.a / (s.a + s.b))[-1, 0])
    assert abs(ms - switch[0]) < 0.1 or abs(ms - switch[1]) < 0.1
    assert ru.free_energy.shape == (10, 1) and len(ru.posteriors["w"]) == 2 and ru.posteriors["w"][0].a.shape == (10, 1)
