"""rxg_binomial_polya_vmp_f32 on the GPU, on both kernels (RXG_OPT_POLYA_PATH = 1 thread per chain, 2 chain groups):
every chain gated against the fp64 reference of test_binomial.py, which gets the fp32-rounded prior: the mean at
TOL_MEAN and the covariance at TOL_COV (relative L2 over the iterations), F at 1e-5 relative to max(|F|, 1) and
non-increasing.  Then near-separable and collinear chains beside healthy ones, flagged chains, KeepEach against shorter
KeepLast runs, bit-exact batch reversal and slicing, the C entry's refusals, and the reference test's assertions through
infer with its 20 simulations in one launch."""
import numpy as np
import pytest
import torch

from test_binomial import FE_TOL, gate, random_problem, reference_assertions, reference_on_f32, reference_simulations

pytestmark = pytest.mark.gpu
PATHS = (1, 2)


@pytest.fixture
def pctx(ctx):
    yield ctx
    ctx.set_option("polya_path", 0)


def run(ctx, path, X, y, n, xi0, W0, its, **kw):
    ctx.set_option("polya_path", path)
    dev = lambda a, t: None if a is None else torch.as_tensor(np.ascontiguousarray(a), dtype=t, device="cuda:0")
    r = ctx.binomial_polya_vmp(dev(X, torch.float32), dev(y, torch.int32), xi0, W0, ntrials=dev(n, torch.int32),
                               iterations=its, keep_each=kw.pop("keep_each", True), **kw)
    return {k: (v.cpu().numpy() if v is not None else None) for k, v in r.items()}


def check_fe_decreases(case, fe):
    assert (np.diff(fe, axis=0) <= FE_TOL * np.maximum(np.abs(fe[1:]), 1)).all(), f"{case}: F increased"


@pytest.mark.parametrize("path", PATHS)
@pytest.mark.parametrize("p", range(1, 9))
def test_every_chain_against_the_fp64_reference(pctx, path, p):
    worst = {}
    for N in (1, 7, 1000, 10000):
        for bern in (False, True):
            nb = 13 if N < 10000 else 5                  # odd batches: ragged chain groups and warps
            X, y, n, xi0, W0 = random_problem(p, N, nb, seed=1000 * p + N + bern, bernoulli=bern)
            its = 6 if N == 10000 else 15
            r = run(pctx, path, X, y, n, xi0, W0, its)
            case = f"path={path} p={p} N={N} bernoulli={bern}"
            for k, v in gate(case, r, reference_on_f32(X, y, n, xi0, W0, its)).items():
                worst[k] = max(worst.get(k, 0.0), v)
            assert (r["status"] == 0).all()
            check_fe_decreases(case, r["free_energy"])
            np.testing.assert_array_equal(r["beta_mean"], r["hist_mean"][-1])
            np.testing.assert_array_equal(r["beta_cov"], r["hist_cov"][-1])
    print(f"worst path={path} p={p}", {k: f"{v:.3g}" for k, v in sorted(worst.items())})


@pytest.mark.parametrize("path", PATHS)
def test_near_separable_and_collinear_chains_beside_healthy_ones(pctx, path):
    X, y, n, xi0, W0 = random_problem(3, 500, 9, seed=21)
    X[:, 1, 2] = X[:, 0, 2]                                      # chain 2: two identical features
    s = np.sign(X[:, 0, 5])                                      # chain 5: y = n exactly where x_0 > 0
    y[:, 5] = np.where(s > 0, n[:, 5], 0)
    r = run(pctx, path, X, y, n, xi0, W0, 30)
    gate(f"path={path}", r, reference_on_f32(X, y, n, xi0, W0, 30))
    assert (r["status"] == 0).all()
    check_fe_decreases(f"path={path}", r["free_energy"])


@pytest.mark.parametrize("path", PATHS)
def test_bad_chains_are_flagged_without_touching_their_neighbours(pctx, path):
    X, y, n, xi0, W0 = random_problem(2, 300, 11, seed=22)
    clean = run(pctx, path, X, y, n, xi0, W0, 10)
    y[17, 3] = n[17, 3] + 1
    X[40, 1, 8] = np.nan
    r = run(pctx, path, X, y, n, xi0, W0, 10)
    assert r["status"].tolist() == [0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0]
    ok = [b for b in range(11) if b not in (3, 8)]
    for k in ("hist_mean", "hist_cov", "free_energy"):
        np.testing.assert_array_equal(r[k][..., ok], clean[k][..., ok])
    n2 = n.copy()
    n2[17, 3], n2[40, 8] = 0, 0
    gate("flagged", r, reference_on_f32(np.nan_to_num(X), np.minimum(y, n2), n2, xi0, W0, 10), chains=[3, 8])


@pytest.mark.parametrize("path", PATHS)
def test_keep_each_entry_k_is_a_k_plus_one_iteration_run(pctx, path):
    X, y, n, xi0, W0 = random_problem(4, 700, 10, seed=23)
    r = run(pctx, path, X, y, n, xi0, W0, 6)
    for k in range(6):
        s = run(pctx, path, X, y, n, xi0, W0, k + 1, keep_each=False, want_free_energy=bool(k % 2))
        np.testing.assert_array_equal(r["hist_mean"][k], s["beta_mean"])
        np.testing.assert_array_equal(r["hist_cov"][k], s["beta_cov"])
        if k % 2:
            np.testing.assert_array_equal(r["free_energy"][: k + 1], s["free_energy"])


@pytest.mark.parametrize("path", PATHS)
def test_batch_reversal_and_slicing_are_bit_exact(pctx, path):
    X, y, n, xi0, W0 = random_problem(3, 900, 21, seed=24)
    r = run(pctx, path, X, y, n, xi0, W0, 8)
    rev = run(pctx, path, X[..., ::-1], y[:, ::-1], n[:, ::-1], xi0, W0, 8)
    sl = run(pctx, path, X[..., 5:12], y[:, 5:12], n[:, 5:12], xi0, W0, 8)
    for k in ("hist_mean", "hist_cov", "free_energy", "status"):
        np.testing.assert_array_equal(rev[k][..., ::-1], r[k])
        np.testing.assert_array_equal(sl[k], r[k][..., 5:12])


def test_the_c_entry_refuses_bad_arguments(pctx, rx):
    X, y, n, xi0, W0 = random_problem(2, 10, 3, seed=25)
    with pytest.raises(rx.RxGaussError) as e:
        run(pctx, 0, np.zeros((10, 9, 3), np.float32), y, n, np.zeros(9), np.eye(9), 2)
    assert e.value.code == 6                                     # p = 9: RXG_ERR_UNSUPPORTED
    for bad in (np.array([[1.0, 0.5], [0.4, 1.0]]), np.array([[1.0, 2.0], [2.0, 1.0]]), np.eye(2) * np.nan):
        with pytest.raises(rx.RxGaussError) as e:
            run(pctx, 0, X, y, n, xi0, bad, 2)
        assert e.value.code == 1
    with pytest.raises(rx.RxGaussError) as e:
        run(pctx, 3, X, y, n, xi0, W0, 2)
    assert e.value.code == 1
    with pytest.raises(ValueError):
        run(pctx, 0, X, y[:5], n, xi0, W0, 2)
    with pytest.raises(ValueError):
        run(pctx, 0, X, y, n, xi0, np.eye(3), 2)
    with pytest.raises(ValueError):
        pctx.binomial_polya_vmp(torch.zeros(10, 2, 3, device="cuda:0"), torch.zeros(10, 3, device="cuda:0"), xi0, W0)


def test_the_reference_assertions_through_infer_in_one_launch(ctx, rx):
    X, y, n, beta = reference_simulations()
    model = rx.binomial_regression(np.zeros(2), np.eye(2))
    data = {"X": X.transpose(2, 0, 1), "y": y.T, "n_trials": n.T}
    launches = ctx.launches
    res = rx.infer(model=model, data=data, iterations=100, free_energy=True, returnvars=rx.KeepEach(),
                   options={"limit_stack_depth": 100}, context=ctx)
    assert ctx.launches == launches + 1
    post = res.posteriors["β"]
    mean, cov = post.mu[-1].cpu().numpy(), post.Sigma[-1].cpu().numpy()
    fes = res.free_energy.cpu().numpy()
    reference_assertions(mean, np.stack([cov[0, 0], cov[1, 1]]), fes, beta)
    gate("infer", {"hist_mean": post.mu.cpu().numpy(), "hist_cov": post.Sigma.cpu().numpy(), "free_energy": fes},
         reference_on_f32(X, y, n, np.zeros(2), np.eye(2), 100))
    one = rx.infer(model=model, data={k: v[4] for k, v in data.items()}, iterations=100, free_energy=True, context=ctx)
    np.testing.assert_allclose(one.posteriors["β"].mu.cpu().numpy(), mean[:, 4], rtol=1e-5)
    bern = rx.infer(model=model, data={"X": data["X"], "y": (y.T > n.T / 2).astype(np.int32)}, iterations=5, context=ctx)
    assert bern.posteriors["β"].mu.shape == (2, 20)
    bad = dict(data, y=data["y"].copy())
    bad["y"][2, 3] = -1
    with pytest.raises(rx.RxGaussError):
        rx.infer(model=model, data=bad, iterations=3, context=ctx)
