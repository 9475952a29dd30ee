"""rxg_gamma_mixture_vmp_f32 on the GPU: every chain gated against the fp64 reference (oracle/gamma_mixture.py) on the
same fp32-rounded inputs.  Per chain: a_hat, the q(b) parameters and q(s) at TOL_MEAN (relative L2 over the components),
the KeepEach histories at 3 TOL_MEAN (over every iteration), the last F at 1e-5 relative to max(|F|, 1) and every earlier
one at 3e-5, q(z) at 1e-3 absolute.  The histories' wider gates follow DESIGN 3.17: the middle iterates of a slowly
converging chain amplify the fp32 rounding of the responsibilities (measured worst 1.12e-5 on F, DESIGN 3.24).  Bit-exact relations with torch.equal; F non-increasing; bad data flag only their chain; the reference
test's call through ``infer`` on its replayed data."""
import numpy as np
import pytest
import torch

from oracle import gamma_mixture as og
from test_gamma_mixture import KEYS, f32, problem, reference_assertions, reference_data, reference_model
from util import TOL_MEAN

pytestmark = pytest.mark.gpu
NB = 7                                         # odd batch
FE_TOL = 1e-5
Z_TOL = 1e-3
GATES = dict(alpha=TOL_MEAN, a_hat=TOL_MEAN, b_shape=TOL_MEAN, b_rate=TOL_MEAN, hist_a=3 * TOL_MEAN,
             hist_b_shape=3 * TOL_MEAN, hist_b_rate=3 * TOL_MEAN)


def dev(a):
    return torch.as_tensor(np.asarray(a, np.float32), device="cuda:0").contiguous()


def run(ctx, y, pri, its, **kw):
    """CUDA and fp64 reference on the same fp32-rounded inputs."""
    p32 = {k: f32(v) for k, v in pri.items()}
    r = ctx.gamma_mixture_vmp(dev(y), *(p32[k] for k in KEYS), iterations=its, want_z=True, keep_each=True, **kw)
    ref = og.gamma_mixture(f32(y), **p32, iterations=its)
    return r, ref


def gate(case, r, ref):
    assert int(r["status"].abs().sum()) == 0 and ref["converged"].all(), case
    for k, tol in GATES.items():
        got = r[k].cpu().numpy().astype(np.float64)
        ax = tuple(range(got.ndim - 1))
        err = np.sqrt(((got - ref[k]) ** 2).sum(ax)) / np.sqrt((ref[k] ** 2).sum(ax))
        assert err.max() < tol, f"{case}: {k} worst chain {int(err.argmax())} err {err.max():.3g} > {tol}"
    ez = np.abs(r["z_prob"].cpu().numpy() - ref["z_prob"]).max()
    assert ez < Z_TOL, f"{case}: z_prob {ez:.3g}"
    fe = r["free_energy"].cpu().numpy()
    efe = np.abs(fe - ref["free_energy"]) / np.maximum(np.abs(ref["free_energy"]), 1.0)
    assert efe[-1].max() < FE_TOL, f"{case}: last free energy {efe[-1].max():.3g}"
    assert efe.max() < 3 * FE_TOL, f"{case}: free energy history {efe.max():.3g}"
    return fe


@pytest.mark.parametrize("K", [2, 3, 5, 8])
def test_every_chain_against_the_fp64_reference(ctx, K):
    for N in (1, 7, 250):
        for its in (1, 50):
            overlap = (N + its) % 2 == 0                 # separated and overlapping components
            y, pri = problem(K, N, NB, seed=1000 * K + N + its, overlap=overlap)
            r, ref = run(ctx, y, pri, its)
            fe = gate(f"K={K} N={N} its={its} overlap={overlap}", r, ref)
            slack = 2 * FE_TOL * np.maximum(np.abs(fe[:-1]), 1.0)
            assert np.all(np.diff(fe, axis=0) <= slack), (K, N, its)


def test_batch_reversal_and_slices_are_bit_exact(ctx):
    y, pri = problem(5, 300, 9, seed=5)
    args = [f32(pri[k]) for k in KEYS]
    yd = dev(y)
    full = ctx.gamma_mixture_vmp(yd, *args, iterations=12, want_z=True, keep_each=True)
    rev = ctx.gamma_mixture_vmp(yd.flip(-1).contiguous(), *args, iterations=12, want_z=True, keep_each=True)
    part = ctx.gamma_mixture_vmp(yd[..., 3:5].contiguous(), *args, iterations=12, want_z=True, keep_each=True)
    for k, v in full.items():
        assert torch.equal(rev[k].flip(-1), v), k
        assert torch.equal(part[k], v[..., 3:5]), k
    lean = ctx.gamma_mixture_vmp(yd, *args, iterations=12, want_free_energy=False)      # optional outputs change nothing
    for k in ("alpha", "a_hat", "b_shape", "b_rate", "status"):
        assert torch.equal(lean[k], full[k]), k
    assert torch.equal(full["hist_a"][-1], full["a_hat"]) and torch.equal(full["hist_b_rate"][-1], full["b_rate"])


def test_a_bad_datum_flags_only_its_chain(ctx):
    from rxinfer_jl_b200 import _lib as L
    y, pri = problem(3, 50, NB, seed=8)
    args = [f32(pri[k]) for k in KEYS]
    good = ctx.gamma_mixture_vmp(dev(y), *args, iterations=5, want_z=True, keep_each=True)
    y[10, 4] = -0.5
    y[3, 1] = np.nan
    bad = ctx.gamma_mixture_vmp(dev(y), *args, iterations=5, want_z=True, keep_each=True)
    assert bad["status"].tolist() == [0, L.RXG_ERR_BAD_ARG, 0, 0, L.RXG_ERR_BAD_ARG, 0, 0]
    keep = [0, 2, 3, 5, 6]
    for k, v in bad.items():
        if k != "status":
            assert torch.equal(v[..., keep], good[k][..., keep]), k
            assert bool(torch.isnan(v[..., [1, 4]]).all()), k


def test_refusals(ctx):
    from rxinfer_jl_b200 import _lib as L
    U, BAD = L.RXG_ERR_UNSUPPORTED, L.RXG_ERR_BAD_ARG
    y = dev(np.ones((4, 3)))
    args = lambda K, **over: [np.asarray(over.get(k, np.ones(K))) for k in KEYS]

    def code(*a, **k):
        with pytest.raises(L.RxGaussError) as e:
            ctx.gamma_mixture_vmp(*a, **k)
        return e.value.code
    assert int(ctx.gamma_mixture_vmp(y, *args(3))["status"].abs().sum()) == 0
    assert code(y, *args(1)) == U and code(y, *args(9)) == U
    assert code(y, *args(3, a_shape0=np.array([1.0, 0.9, 1.0]))) == U
    assert code(dev(np.ones((0, 3))), *args(3)) == BAD
    assert code(y, *args(3), iterations=0) == BAD
    for k in KEYS:
        for v in (0.0, -1.0, np.nan, np.inf):
            assert code(y, *args(3, **{k: np.array([1.0, v, 1.0])})) == BAD, (k, v)
    with pytest.raises(ValueError):
        ctx.gamma_mixture_vmp(dev(np.ones((4, 2, 3))), *args(3))


def test_infer_runs_the_reference_test(ctx, rx):
    """gamma_mixture_tests.jl:59-94 through infer on the replayed data: KeepEach lengths, E[q(s)], the component means;
    the free energy against the fp64 reference (the reference's pin is not reproduced by any data reading, DESIGN 3.24)."""
    y, mixing = reference_data()
    model, cons, init = reference_model(mixing)
    res = rx.infer(model=model, data={"y": y}, constraints=cons, initialization=init, free_energy=True, iterations=50,
                   returnvars={"s": rx.KeepLast(), "z": rx.KeepLast(), "as": rx.KeepEach(), "bs": rx.KeepEach()},
                   context=ctx)
    assert len(res.posteriors["as"]) == 2 and res.posteriors["as"][0].value.shape == (50,)
    assert len(res.posteriors["bs"]) == 2 and res.posteriors["bs"][1].a.shape == (50,)
    assert res.free_energy.shape == (50,) and res.posteriors["z"].p.shape == (250, 2)
    a_hat = np.array([float(q.mean()[-1]) for q in res.posteriors["as"]])
    b_mean = np.array([float(q.mean()[-1]) for q in res.posteriors["bs"]])
    alpha = res.posteriors["s"].alpha.cpu().numpy()
    reference_assertions(a_hat, b_mean, alpha / alpha.sum())
    from rxinfer_jl_b200.inference import gamma_mixture_arguments
    arr = gamma_mixture_arguments(model, cons, init)
    ref = og.gamma_mixture(f32(y)[:, None], **{k: f32(v) for k, v in arr.items()}, iterations=50)
    fe = res.free_energy.cpu().numpy()
    assert np.abs(fe - ref["free_energy"][:, 0]).max() < FE_TOL * np.abs(ref["free_energy"]).max()
    # KeepLast everywhere: the last iteration of the KeepEach results, bit for bit
    last = rx.infer(model=model, data={"y": y}, constraints=cons, initialization=init, iterations=50, context=ctx)
    assert torch.equal(last.posteriors["as"][0].value, res.posteriors["as"][0].value[-1])
    assert torch.equal(last.posteriors["bs"][1].b, res.posteriors["bs"][1].b[-1])
    assert last.free_energy is None
    # a flagged chain raises
    with pytest.raises(rx.RxGaussError):
        rx.infer(model=model, data={"y": np.stack([y, -y], -1)}, constraints=cons, initialization=init, iterations=3,
                 context=ctx)
