"""rxg_hgf_vmp_learn_f32 on the GPU: every chain gated against the fp64 reference of test_hgf_learn.py, which gets the
fp32-rounded inputs, over T in {1, 2, 7, 300, 1000}, {1, 20} iterations and three hyper-parameter sets (test_hgf_learn.gate:
q(x), q(z) at TOL_MEAN / TOL_COV, q(kappa), q(omega) and their KeepEach histories at the stated bounds, the free energy at
1e-5 relative to max(|F|, 1)).  Then T = 10 000 at the same bounds, an odd batch with half the steps missing, batch reversal bit for bit, the
KeepEach final slot against the KeepLast output, a chain with infinite data beside healthy ones (also through infer, which
returns the flags), the reference test's assertions through infer, and every refusal of the C entry."""
import ctypes

import numpy as np
import pytest
import torch

from test_hgf_learn import DEFAULT, HYPER, SET_B, SET_C, gate, hgf1_assertions, reference_data, reference_on_f32, series

pytestmark = pytest.mark.gpu
NB = 7                                         # odd batch


def run(ctx, y, its, h, keep_each=True, want_free_energy=True):
    r = ctx.hgf_vmp_learn(torch.as_tensor(np.asarray(y, np.float32), device="cuda:0").contiguous(), **h, iterations=its,
                          keep_each=keep_each, want_free_energy=want_free_energy)
    return {k: (v.cpu().numpy() if v is not None else None) for k, v in r.items()}


@pytest.mark.parametrize("hyper", sorted(HYPER))
def test_every_chain_against_the_fp64_reference(ctx, hyper):
    h = HYPER[hyper]
    for T in (1, 2, 7, 300, 1000):
        for its in (1, 20):
            y = series(T, NB, seed=7 * T + its, p_missing=0.2 if T > 2 else 0.0)
            gate(f"{hyper} T={T} its={its}", run(ctx, y, its, h), reference_on_f32(y, its, h))


def test_long_series(ctx):
    """T = 10 000; a chain on which the reference's GH products collapse must be the one flagged (gate)."""
    y = series(10000, 3, seed=77, p_missing=0.1)
    gate("T=10000", run(ctx, y, 5, SET_C), reference_on_f32(y, 5, SET_C))


def test_half_the_steps_missing_odd_batch(ctx):
    y = series(400, 9, seed=78, p_missing=0.5)
    gate("half missing", run(ctx, y, 10, SET_B), reference_on_f32(y, 10, SET_B))


def test_batch_reversal_is_bit_exact_and_keep_each_ends_in_keep_last(ctx):
    y = series(300, 33, seed=79, p_missing=0.2)
    a = run(ctx, y, 8, SET_B)
    b = run(ctx, y[:, ::-1].copy(), 8, SET_B)
    for k in ("xz", "x0", "kw", "hist_kw", "free_energy", "status"):
        assert np.array_equal(a[k], b[k][..., ::-1]), k
    yy = torch.as_tensor(np.asarray(y, np.float32), device="cuda:0").contiguous()
    each = ctx.hgf_vmp_learn(yy, **SET_B, iterations=8, keep_each=True)
    last = ctx.hgf_vmp_learn(yy, **SET_B, iterations=8, keep_each=False, want_free_energy=False)
    assert torch.equal(each["hist_kw"][-1], last["kw"]) and torch.equal(each["kw"], last["kw"])
    assert torch.equal(each["xz"], last["xz"]) and torch.equal(each["x0"], last["x0"])


def test_infinite_data_flags_its_chain_only(ctx):
    y = series(50, 5, seed=80, p_missing=0.1)
    y[20, 3] = np.inf
    r = run(ctx, y, 4, SET_C)
    assert list(r["status"]) == [0, 0, 0, 5, 0]
    keep = [0, 1, 2, 4]
    gate("neighbours of an inf chain", {k: (v[..., keep] if v is not None else None) for k, v in r.items()},
         reference_on_f32(y[:, keep], 4, SET_C))


def test_infer_returns_flagged_chains_beside_the_others(ctx, rx):
    """A chain flagged RXG_ERR_NAN does not make infer raise: result.status names it and the other chains' posteriors are
    those of the C entry."""
    from rxinfer_jl_b200 import MeanField, NormalMeanVariance, hgf_offline
    y = series(50, 5, seed=80, p_missing=0.1)
    y[20, 3] = np.inf
    h = SET_C
    p, i = h["prior"], h["init"]
    model = hgf_offline(κ_prior=p[0:2], ω_prior=p[2:4], x0_prior=p[4:6], z1_prior=p[6:8], z_precision=h["z_precision"],
                        y_variance=h["y_variance"])
    init = {k: NormalMeanVariance(*i[2 * j:2 * j + 2]) for j, k in enumerate(("κ", "ω", "z", "x"))}
    res = rx.infer(model=model, data={"y": torch.as_tensor(y, dtype=torch.float32)}, constraints=MeanField(),
                   initialization=init, iterations=4, free_energy=True)
    assert res.status.cpu().tolist() == [0, 0, 0, 5, 0]
    r = run(ctx, y, 4, h)
    keep = [0, 1, 2, 4]
    assert np.array_equal(res.posteriors["x"].m.cpu().numpy()[:, keep], r["xz"][:, 0, keep])
    assert np.array_equal(res.posteriors["κ"].v.cpu().numpy()[keep], r["kw"][0, 1, keep])
    assert np.array_equal(res.free_energy.cpu().numpy()[:, keep], r["free_energy"][:, keep])


def test_reference_configuration_through_infer(rx):
    from rxinfer_jl_b200 import KeepEach, KeepLast, MeanField, NormalMeanVariance, hgf_offline
    y = reference_data()
    init = {"κ": NormalMeanVariance(1.0, 1.0), "ω": NormalMeanVariance(0.0, 1.0), "z": NormalMeanVariance(0.0, 1.0),
            "x": NormalMeanVariance(0.0, 1.0)}
    res = rx.infer(model=hgf_offline(), data={"y": torch.as_tensor(y, dtype=torch.float32)}, constraints=MeanField(),
                   initialization=init, iterations=10, free_energy=True,
                   returnvars={"x": KeepLast(), "z": KeepLast(), "κ": KeepEach(), "ω": KeepEach()})
    x = res.posteriors["x"]
    hgf1_assertions(x.m.cpu().numpy(), x.v.cpu().numpy(), res.free_energy.cpu().numpy())
    ref = reference_on_f32(y, 10, DEFAULT)
    r = {"xz": torch.stack([x.m, x.v, res.posteriors["z"].m, res.posteriors["z"].v], 1).cpu().numpy(),
         "x0": torch.stack([res.posteriors["x_0"].m, res.posteriors["x_0"].v]).cpu().numpy(),
         "hist_kw": torch.stack([torch.stack([res.posteriors[n].m, res.posteriors[n].v], 1) for n in ("κ", "ω")], 1).cpu().numpy(),
         "free_energy": res.free_energy.cpu().numpy(), "status": np.zeros(1, np.int32)}
    gate("hgf_1 through infer", r, ref)
    assert res.posteriors["κ"].m.shape == (10, 1)


def test_every_refusal_of_the_c_entry(ctx, rx):
    L = rx._lib
    lib = ctx.lib
    T, nb = 5, 3
    y = torch.zeros(T, nb, device="cuda:0")
    xz, x0, kw = torch.empty(T, 4, nb, device="cuda:0"), torch.empty(2, nb, device="cuda:0"), torch.empty(2, 2, nb, device="cuda:0")
    fp = lambda t: L.as_fp(t.data_ptr()) if t is not None else L.as_fp(0)
    arr = lambda v: np.asarray(v, np.float32)
    null_d = ctypes.cast(ctypes.c_void_p(None), ctypes.POINTER(ctypes.c_double))
    null_i = ctypes.cast(ctypes.c_void_p(None), L.i32p)
    good_p, good_i = arr(DEFAULT["prior"]), arr(DEFAULT["init"])

    def call(T=T, nb=nb, its=2, prior=good_p, zp=1.0, yv=1.0, init=good_i, yy=y, out=xz, k=kw, flags=L.PTR_DEVICE):
        return lib.rxg_hgf_vmp_learn_f32(ctx.h, T, nb, its, prior.ctypes.data_as(L.fp) if prior is not None else L.as_fp(0),
                                         zp, yv, init.ctypes.data_as(L.fp) if init is not None else L.as_fp(0), fp(yy),
                                         fp(x0), fp(out), fp(k), L.as_fp(0), null_d, null_i, flags)

    assert call() == L.RXG_OK
    bad = dict(T=0, nb=0, its=0, zp=0.0, yv=-1.0, prior=None, init=None, yy=None, out=None, k=None)
    for k, v in bad.items():
        assert call(**{k: v}) == L.RXG_ERR_BAD_ARG, k
    assert call(zp=float("nan")) == L.RXG_ERR_BAD_ARG
    for i in (1, 3, 5, 7):
        p = good_p.copy(); p[i] = 0.0
        assert call(prior=p) == L.RXG_ERR_BAD_ARG, ("prior", i)
        q = good_i.copy(); q[i] = -1.0
        assert call(init=q) == L.RXG_ERR_BAD_ARG, ("init", i)
    p = good_p.copy(); p[0] = np.inf
    assert call(prior=p) == L.RXG_ERR_BAD_ARG
    assert call(flags=0) == L.RXG_ERR_UNSUPPORTED
    assert lib.rxg_hgf_vmp_learn_f32(None, T, nb, 2, good_p.ctypes.data_as(L.fp), 1.0, 1.0, good_i.ctypes.data_as(L.fp),
                                     fp(y), fp(x0), fp(xz), fp(kw), L.as_fp(0), null_d, null_i, L.PTR_DEVICE) == L.RXG_ERR_BAD_ARG
