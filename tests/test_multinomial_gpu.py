"""rxg_multinomial_polya_vmp_f32 / rxg_multinomial_polya_online_f32 on the GPU: every chain gated against the fp64
reference of test_multinomial.py, which gets the fp32-rounded prior (the mean at TOL_MEAN and the covariance at TOL_COV,
relative L2 over the iterations or data, F at 1e-5 relative to max(|F|, 1)) across K, trials and sample counts; padding
with all-zero samples equals dropping them, bit for bit; flagged chains leave their neighbours' bits alone; KeepEach
entry k is a (k + 1)-iteration run; batch reversal and slicing are bit-exact; online over T = 5000 at K = 40 against the
reference, uneven chunks and the in-place carry bit-identical to one call; the C entries' refusals; and both items of the
reference test through infer."""
import numpy as np
import pytest
import torch

from test_multinomial import (FE_TOL, OFFLINE_CONVERGED, OFFLINE_MSE_PASS, OFFLINE_SEEDS, gate, offline_assertions,
                              online_reference_on_f32, random_problem, reference_offline, reference_on_f32,
                              reference_online)
from oracle import multinomial as om

pytestmark = pytest.mark.gpu
DEVICE_SLACK = 1e-11     # relative round-off of the device's F near convergence (offline_assertions)


def dev(a, t=torch.int32):
    return None if a is None else torch.as_tensor(np.ascontiguousarray(a), dtype=t, device="cuda:0")


def host(r):
    return {k: (v.cpu().numpy() if isinstance(v, torch.Tensor) else v) for k, v in r.items()}


def run(ctx, y, xi0, W0, its, **kw):
    return host(ctx.multinomial_polya_vmp(dev(y), xi0, W0, iterations=its, keep_each=kw.pop("keep_each", True), **kw))


def run_online(ctx, y, xi0, W0, its=1, **kw):
    return host(ctx.multinomial_polya_online(dev(y), xi0, W0, iterations=its, **kw))


@pytest.mark.parametrize("K", [2, 3, 5, 10, 17, 33, 40, 64])
def test_every_chain_against_the_fp64_reference(ctx, K):
    worst = {}
    for n, trials in ((1, 20), (50, 3), (1000, 20), (1000, 500)):
        nb = 13 if n < 1000 else 5                        # odd batches: ragged CTAs
        y, xi0, W0 = random_problem(K, n, nb, seed=1000 * K + n + trials, max_trials=trials)
        its = 12
        r = run(ctx, y, xi0, W0, its)
        case = f"K={K} n={n} trials={trials}"
        for k, v in gate(case, r, reference_on_f32(y, xi0, W0, its)).items():
            worst[k] = max(worst.get(k, 0.0), v)
        assert (r["status"] == 0).all()
        assert (np.diff(r["free_energy"], axis=0) <= FE_TOL * np.maximum(np.abs(r["free_energy"][1:]), 1)).all(), case
        np.testing.assert_array_equal(r["psi_mean"], r["hist_mean"][-1])
        np.testing.assert_array_equal(r["psi_cov"], r["hist_cov"][-1])
    print(f"worst K={K}", {k: f"{v:.3g}" for k, v in sorted(worst.items())})


def test_padding_with_all_zero_samples_equals_dropping_them(ctx):
    y, xi0, W0 = random_problem(10, 300, 9, seed=21)
    short = run(ctx, y[:200], xi0, W0, 8)
    pad = y.copy()
    pad[200:] = 0
    r = run(ctx, pad, xi0, W0, 8)
    for k in ("hist_mean", "hist_cov", "free_energy", "status"):
        np.testing.assert_array_equal(r[k], short[k])


def test_flagged_chains_leave_their_neighbours_alone(ctx):
    y, xi0, W0 = random_problem(6, 300, 11, seed=22)
    clean = run(ctx, y, xi0, W0, 10)
    bad = y.copy()
    bad[17, 2, 3] = -1
    bad[40, 5, 8] = -7
    r = run(ctx, bad, xi0, W0, 10)
    assert r["status"].tolist() == [0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0]
    ok = [b for b in range(11) if b not in (3, 8)]
    for k in ("hist_mean", "hist_cov", "free_energy"):
        np.testing.assert_array_equal(r[k][..., ok], clean[k][..., ok])
    zeroed = y.copy()
    zeroed[17, :, 3] = 0
    zeroed[40, :, 8] = 0
    gate("flagged", r, reference_on_f32(zeroed, xi0, W0, 10), chains=[3, 8])
    o = run_online(ctx, bad[:60], xi0, W0)
    assert o["status"].tolist() == r["status"].tolist()
    oc = run_online(ctx, y[:60], xi0, W0)
    for k in ("hist_mean", "free_energy", "m", "S"):
        np.testing.assert_array_equal(o[k][..., ok], oc[k][..., ok])


def test_keep_each_entry_k_is_a_k_plus_one_iteration_run(ctx):
    y, xi0, W0 = random_problem(8, 700, 10, seed=23)
    r = run(ctx, y, xi0, W0, 6)
    for k in range(6):
        s = run(ctx, y, xi0, W0, k + 1, keep_each=False, want_free_energy=bool(k % 2))
        np.testing.assert_array_equal(r["hist_mean"][k], s["psi_mean"])
        np.testing.assert_array_equal(r["hist_cov"][k], s["psi_cov"])
        if k % 2:
            np.testing.assert_array_equal(r["free_energy"][: k + 1], s["free_energy"])


def test_batch_reversal_and_slicing_are_bit_exact(ctx):
    y, xi0, W0 = random_problem(12, 900, 21, seed=24)
    r = run(ctx, y, xi0, W0, 8)
    rev = run(ctx, y[..., ::-1], xi0, W0, 8)
    sl = run(ctx, y[..., 5:12], xi0, W0, 8)
    for k in ("hist_mean", "hist_cov", "free_energy", "status"):
        np.testing.assert_array_equal(rev[k][..., ::-1], r[k])
        np.testing.assert_array_equal(sl[k], r[k][..., 5:12])
    o = run_online(ctx, y[:200], xi0, W0)
    orev = run_online(ctx, y[:200, :, ::-1], xi0, W0)
    for k in ("hist_mean", "hist_cov", "free_energy", "m", "S"):
        np.testing.assert_array_equal(orev[k][..., ::-1], o[k])


def test_online_over_5000_data_against_the_reference_and_chunked_bit_for_bit(ctx):
    y1, W, _ = reference_online()
    rng = np.random.default_rng(25)
    y = np.stack([y1] + [reference_online(seed=s)[0] for s in (1, 2)], -1)       # [5000, 40, 3]
    xi0 = 0.1 * rng.standard_normal(39)
    whole = run_online(ctx, y, xi0, W)
    ref = online_reference_on_f32(y[..., :2], xi0, W)
    worst = gate("online T=5000 K=40", {k: whole[k][..., :2] for k in ("hist_mean", "hist_cov", "free_energy")}, ref)
    print("worst online", {k: f"{v:.3g}" for k, v in sorted(worst.items())})
    assert (whole["status"] == 0).all()
    m = S = None
    parts = []
    for a, b in ((0, 1), (1, 2), (2, 777), (777, 778), (778, 5000)):
        o = run_online(ctx, y[a:b], xi0, W, m=m, S=S)
        m, S = dev(o["m"], torch.float64), dev(o["S"], torch.float64)
        parts.append(o)
    for k in ("hist_mean", "hist_cov", "free_energy"):
        np.testing.assert_array_equal(np.concatenate([p[k] for p in parts]), whole[k])
    np.testing.assert_array_equal(m.cpu().numpy(), whole["m"])
    np.testing.assert_array_equal(S.cpu().numpy(), whole["S"])
    first = ctx.multinomial_polya_online(dev(y[:1000]), xi0, W)
    mi, Si = first["m"], first["S"]
    r = ctx.multinomial_polya_online(dev(y[1000:]), xi0, W, m=mi, S=Si, in_place=True, keep_cov=False)
    assert r["m"].data_ptr() == mi.data_ptr() and r["hist_cov"] is None
    np.testing.assert_array_equal(mi.cpu().numpy(), whole["m"])
    np.testing.assert_array_equal(Si.cpu().numpy(), whole["S"])
    np.testing.assert_array_equal(r["free_energy"].cpu().numpy(), whole["free_energy"][1000:])


def test_online_iterations_against_the_reference(ctx):
    y, xi0, W0 = random_problem(20, 80, 4, seed=26)
    for its in (2, 5):
        gate(f"online its={its}", run_online(ctx, y, xi0, W0, its), online_reference_on_f32(y, xi0, W0, its))


def test_the_c_entries_refuse_bad_arguments(ctx, rx):
    y, xi0, W0 = random_problem(4, 10, 3, seed=27)
    for K in (1, 65):
        with pytest.raises(rx.RxGaussError) as e:
            run(ctx, np.zeros((10, K, 3), np.int32), np.zeros(K - 1), np.eye(K - 1), 2)
        assert e.value.code == 6                                 # RXG_ERR_UNSUPPORTED
        with pytest.raises(rx.RxGaussError) as e:
            run_online(ctx, np.zeros((10, K, 3), np.int32), np.zeros(K - 1), np.eye(K - 1))
        assert e.value.code == 6
    for bad in (np.array([[1.0, 0.5, 0], [0.4, 1.0, 0], [0, 0, 1]]), np.diag([1.0, -1.0, 1.0]), np.eye(3) * np.nan):
        with pytest.raises(rx.RxGaussError) as e:
            run(ctx, y, xi0, bad, 2)
        assert e.value.code == 1
        with pytest.raises(rx.RxGaussError) as e:
            run_online(ctx, y, xi0, bad)
        assert e.value.code == 1
    with pytest.raises(ValueError):
        run(ctx, y, xi0, np.eye(4), 2)
    with pytest.raises(ValueError):
        ctx.multinomial_polya_vmp(dev(y, torch.float32), xi0, W0)
    with pytest.raises(ValueError):
        run_online(ctx, y, xi0, W0, m=torch.zeros(3, 3, dtype=torch.float64, device="cuda:0"))


def test_the_offline_reference_item_through_infer(ctx, rx):
    """multinomialreg_tests.jl, offline: 20 seeded data sets in one call; F[end] < F[1] and F[end] <= F[end-1] on every
    one; the mse and convergence assertions hold on the same data sets as on the fp64 reference."""
    data = [reference_offline(s) for s in OFFLINE_SEEDS]
    W = data[0][1]                   # one prior for the batch (the C entry shares it); the fp64 reference gets it too
    y = np.stack([d[0] for d in data])
    model = rx.multinomial_regression(np.zeros(9), W)
    launches = ctx.launches
    res = rx.infer(model=model, data={"y": y}, iterations=100, free_energy=True, returnvars=rx.KeepLast(),
                   options={"limit_stack_depth": 100}, context=ctx)
    assert ctx.launches == launches + 2                          # the data pass and the iterations
    mean = res.posteriors["ψ"].mu.cpu().numpy()
    fes = res.free_energy.cpu().numpy()
    ref = reference_on_f32(y.transpose(1, 2, 0), np.zeros(9), W, 100)
    gate("offline item", {"hist_mean": mean[None], "free_energy": fes},
         {"hist_mean": ref["hist_mean"][-1:], "free_energy": ref["free_energy"]})
    dev_mse = dev_conv = 0
    for b, (_, _, p) in enumerate(data):
        a = offline_assertions(mean[:, b], fes[:, b], p, slack=DEVICE_SLACK)
        e = offline_assertions(ref["hist_mean"][-1][:, b], ref["free_energy"][:, b], p)
        assert a[0] == e[0], (b, a, e)
        dev_mse += a[0]
        dev_conv += a[1]
    print(f"offline item, shared W: mse < 2e-5 on {dev_mse} of 20, |dF| < 1e-8 on {dev_conv} of 20")
    one = rx.infer(model=rx.multinomial_regression(np.zeros(9), data[3][1]), data={"y": data[3][0]}, iterations=100,
                   free_energy=True, context=ctx)
    r1 = om.vmp(data[3][0], np.zeros(9), np.asarray(data[3][1], np.float32).astype(np.float64), 100)
    np.testing.assert_allclose(one.posteriors["ψ"].mu.cpu().numpy(), r1["mean"][-1], rtol=1e-5, atol=1e-7)
    assert one.free_energy.shape == (100,)
    bad = y.copy()
    bad[2, 3, 0] = -1
    with pytest.raises(rx.RxGaussError):
        rx.infer(model=model, data={"y": bad}, iterations=3, context=ctx)


def test_the_offline_item_seed_by_seed_against_the_reference(ctx):
    """Each seed with its own W_ψ: the mse assertion holds on the same data sets as on the fp64 reference, the last
    free-energy change agrees with the reference's to the step's round-off, and the counts are printed (DESIGN 3.22)."""
    mse_pass = conv = 0
    for seed in OFFLINE_SEEDS:
        y, W, p = reference_offline(seed)
        r = run(ctx, y[..., None], np.zeros(9), W, 100, keep_each=False)
        o = om.vmp(y, np.zeros(9), np.asarray(W, np.float32).astype(np.float64), 100)
        fd, fo = r["free_energy"][:, 0], o["free_energy"]
        a = offline_assertions(r["psi_mean"][:, 0], fd, p, slack=DEVICE_SLACK)
        e = offline_assertions(o["mean"][-1], fo, p)
        assert a[0] == e[0], (seed, a, e)
        assert abs((fd[-2] - fd[-1]) - (fo[-2] - fo[-1])) <= DEVICE_SLACK * abs(fo[-1]), seed
        mse_pass += a[0]
        conv += a[1]
    assert mse_pass == OFFLINE_MSE_PASS
    print(f"offline item per seed: mse < 2e-5 on {mse_pass} of 20, |dF| < 1e-8 on {conv} of 20 "
          f"(reference: {OFFLINE_MSE_PASS}, {OFFLINE_CONVERGED})")


def test_the_online_reference_item_through_infer(ctx, rx):
    """multinomialreg_tests.jl, online: K = 40, N = 50, 5000 data, one iteration per datum; mse < 1e-3 and
    free_energy_final_only_history[end] < [1]; datastream chunks and pushes give the same bits."""
    from rxinfer_jl_b200.distributions import MvNormalWeightedMeanPrecision
    y, W, p = reference_online()
    model = rx.multinomial_regression_online()
    init = {"ψ": MvNormalWeightedMeanPrecision(np.zeros(39), W)}
    eng = rx.infer(model=model, data={"y": y}, initialization=init, iterations=1,
                   autoupdates="ξ_ψ, W_ψ = weightedmean_precision(q(ψ))", keephistory=len(y), free_energy=True,
                   context=ctx)
    assert eng.is_completed and eng.ticks == 5000
    h = eng.history["ψ"]
    m = h.mu[-1][:, 0].cpu().numpy()
    assert np.mean((om.stick_breaking(m) - p) ** 2) < 1e-3
    fe = eng.free_energy_final_only_history.cpu().numpy()
    assert fe.shape == (5000, 1) and fe[-1, 0] < fe[0, 0]
    ref = online_reference_on_f32(y[..., None], np.zeros(39), W)
    gate("online item", {"hist_mean": h.mu.cpu().numpy(), "hist_cov": h.Sigma.cpu().numpy(), "free_energy": fe}, ref)
    yd = dev(y[..., None])
    chunks = [yd[:100], yd[100:101], yd[101:]]
    eng2 = rx.infer(model=model, datastream=chunks, batch=1, initialization=init, autoupdates=True, keephistory=10,
                    free_energy=True, context=ctx)
    assert torch.equal(eng2.history["ψ"].mu, h.mu[-10:])
    assert torch.equal(eng2.free_energy_final_only_history, eng.free_energy_final_only_history)
    eng3 = rx.infer(model=model, datastream=None, batch=1, initialization=init, autoupdates=True, free_energy=True,
                    context=ctx)
    for c in chunks:
        eng3.push(c)
    assert torch.equal(eng3.posteriors["ψ"].mu, eng2.posteriors["ψ"].mu)
    with pytest.raises(RuntimeError):
        eng3.history
    bad = yd[:5].clone()
    bad[2, 0, 0] = -1
    with pytest.raises(rx.RxGaussError):
        eng3.push(bad)
