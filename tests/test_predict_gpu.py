"""GPU parity of rxg_lgssm_smooth_predict_f32: the observation predictions and forecasts against the reference-schedule
oracle (oracle/predict.py), the two kernel routes against each other, the unchanged posteriors, the covariance output
forms, the port of the reference's "Predictions in State Space Models" tests #1 / #1.1 and the argument errors."""
import ctypes

import numpy as np
import pytest
import torch

from oracle.predict import predict_reference_schedule
from util import TOL_COV, TOL_MEAN, rel_l2

pytestmark = pytest.mark.gpu

# conditioning stress (Q = 1e-2 I, P = 1e2 I): the error gate of this case, see DESIGN.md section 5
STRESS_TOL_MEAN = 1e-3


def _model(d, m, seed, batch=None):
    """Random stable model, rounded to fp32 once (shared, or per chain [batch, ...] for the oracle)."""
    rng = np.random.default_rng(seed)

    def one():
        A = 0.95 * np.linalg.qr(rng.standard_normal((d, d)))[0]
        B = rng.standard_normal((m, d)) / np.sqrt(d)
        G = rng.standard_normal((m, m)) / np.sqrt(m)
        return dict(A=A, B=B, P=0.05 * np.eye(d), Q=np.eye(m) + 0.1 * G @ G.T, m0=rng.standard_normal(d),
                    S0=4.0 * np.eye(d), u=0.1 * rng.standard_normal(d))
    ms = [one() for _ in range(batch)] if batch else [one()]
    out = {k: np.stack([x[k] for x in ms]) if batch else ms[0][k] for k in ms[0]}
    return {k: v.astype(np.float32).astype(np.float64) for k, v in out.items()}


def _dev_model(M):
    """[batch, ...] oracle arrays -> device arrays with the batch axis innermost."""
    return {k: torch.tensor(np.ascontiguousarray(np.moveaxis(v, 0, -1)), dtype=torch.float32, device="cuda")
            for k, v in M.items()}


def _run(ctx, d, m, T, batch, H, mask_kind="none", per_chain=False, with_u=True, tf=False, force_per_chain=False, seed=0):
    rng = np.random.default_rng(seed + 1000)
    M = _model(d, m, seed, batch if per_chain else None)
    y = rng.standard_normal((T, m, batch)).astype(np.float32)
    mask = None
    if mask_kind == "shared":
        mask = np.ones(T, dtype=np.uint8)
        mask[0] = 0
        mask[-1] = 0
        if T > 4:
            mask[T // 2] = 0
    elif mask_kind == "per_chain":
        mask = (rng.random((T, batch)) > 0.3).astype(np.uint8)
        mask[-min(3, T):, 0] = 0                 # trailing gap
        if batch > 1:
            mask[:, 1] = 0                        # prior-only chain
    u = M["u"] if with_u else None
    ref = predict_reference_schedule(y, M["A"], M["B"], M["P"], M["Q"], M["m0"], M["S0"], mask, u=u, transition_first=tf,
                                     horizon=H)
    yd = torch.tensor(y, device="cuda")
    dm = None if mask is None else (mask if mask.ndim == 1 else torch.tensor(mask, device="cuda"))
    if force_per_chain and mask is not None and mask.ndim == 1:      # a shared pattern belongs to the table route
        dm = torch.tensor(np.repeat(mask[:, None], batch, axis=1), device="cuda")
    if per_chain:
        D = _dev_model(M)
        args = [D[k] for k in ("A", "B", "P", "Q", "m0", "S0")]
        ud = D["u"] if with_u else None
    else:
        args = [M[k] for k in ("A", "B", "P", "Q", "m0", "S0")]
        ud = u
    r = ctx.lgssm_predict(yd, *args, horizon=H, u=ud, mask=dm, per_chain_model=per_chain, transition_first=tf,
                          force_per_chain_path=force_per_chain, want_status=True)
    torch.cuda.synchronize()
    return r, ref


def _check(r, ref, H):
    assert (r["status"].cpu().numpy() == 0).all()
    assert rel_l2(r["pred_mean"].cpu().numpy(), ref["pred_mean"]) < TOL_MEAN
    assert rel_l2(r["pred_cov"].cpu().numpy(), ref["pred_cov"]) < TOL_COV
    if H:
        assert rel_l2(r["fc_mean"].cpu().numpy(), ref["fc_mean"]) < TOL_MEAN
        assert rel_l2(r["fc_cov"].cpu().numpy(), ref["fc_cov"]) < TOL_COV


SHAPES = [(1, 1), (2, 1), (4, 4), (6, 6), (5, 3), (16, 16), (33, 20), (64, 64)]


@pytest.mark.parametrize("d,m", SHAPES)
def test_shared_model_shared_mask_matches_oracle(ctx, d, m):
    r, ref = _run(ctx, d, m, T=40, batch=37 if d <= 6 else 9, H=17, mask_kind="shared", seed=d * 100 + m)
    _check(r, ref, 17)


@pytest.mark.parametrize("d,m", SHAPES)
def test_per_chain_model_and_mask_matches_oracle(ctx, d, m):
    r, ref = _run(ctx, d, m, T=24, batch=5, H=1, mask_kind="per_chain", per_chain=True, tf=True, seed=d * 10 + m)
    _check(r, ref, 1)


@pytest.mark.parametrize("d,m,T,H,batch", [(4, 4, 1, 0, 16), (4, 4, 2, 1, 16), (16, 16, 1, 17, 4), (2, 1, 2, 0, 33),
                                           (4, 4, 1000, 1, 16), (2, 1, 1100, 17, 16), (4, 4, 1100, 0, 8)])
def test_lengths_and_horizons_match_oracle(ctx, d, m, T, H, batch):
    r, ref = _run(ctx, d, m, T=T, batch=batch, H=H, mask_kind="none", with_u=(T % 2 == 0), tf=(T == 1), seed=T + d)
    _check(r, ref, H)


@pytest.mark.parametrize("d,m", [(4, 4), (2, 1), (5, 3), (16, 16)])
def test_per_chain_path_only_matches_oracle(ctx, d, m):
    r, ref = _run(ctx, d, m, T=30, batch=6, H=3, mask_kind="none", force_per_chain=True, seed=7 + d)
    _check(r, ref, 3)


@pytest.mark.parametrize("d,m,mask_kind", [(4, 4, "none"), (6, 6, "shared"), (33, 20, "none")])
def test_routes_agree(ctx, d, m, mask_kind):
    ra, _ = _run(ctx, d, m, T=50, batch=12, H=5, mask_kind=mask_kind, seed=3)
    rb, _ = _run(ctx, d, m, T=50, batch=12, H=5, mask_kind=mask_kind, seed=3, force_per_chain=True)
    for k, tol in (("pred_mean", TOL_MEAN), ("pred_cov", TOL_COV), ("fc_mean", TOL_MEAN), ("fc_cov", TOL_COV)):
        assert rel_l2(ra[k].cpu().numpy(), rb[k].cpu().numpy()) < tol, k


@pytest.mark.parametrize("d,m,mask_kind,per_chain", [(4, 4, "none", False), (16, 16, "none", False), (5, 3, "shared", False),
                                                     (4, 4, "per_chain", True)])
def test_posteriors_are_bitwise_those_of_the_smoother(ctx, d, m, mask_kind, per_chain):
    T, batch = 60, 40
    rng = np.random.default_rng(5)
    M = _model(d, m, 11, batch if per_chain else None)
    y = torch.tensor(rng.standard_normal((T, m, batch)).astype(np.float32), device="cuda")
    mask = None
    if mask_kind == "shared":
        mask = np.ones(T, dtype=np.uint8); mask[::7] = 0
    elif mask_kind == "per_chain":
        mask = torch.tensor((rng.random((T, batch)) > 0.2).astype(np.uint8), device="cuda")
    if per_chain:
        D = _dev_model(M)
        args, u = [D[k] for k in ("A", "B", "P", "Q", "m0", "S0")], D["u"]
    else:
        args, u = [M[k] for k in ("A", "B", "P", "Q", "m0", "S0")], M["u"]
    s = ctx.lgssm(y, *args, u=u, mask=mask, want_evidence=True, per_chain_model=per_chain)
    p = ctx.lgssm_predict(y, *args, horizon=4, u=u, mask=mask, want_evidence=True, per_chain_model=per_chain)
    torch.cuda.synchronize()
    for k in ("mean", "cov", "neg_log_evidence"):
        assert torch.equal(s[k], p[k]), k


@pytest.mark.parametrize("d,m", [(4, 4), (16, 16)])
def test_shared_covariance_tables_and_means_only(ctx, d, m):
    T, batch, H = 70, 50, 6
    M = _model(d, m, 21)
    rng = np.random.default_rng(9)
    y = torch.tensor(rng.standard_normal((T, m, batch)).astype(np.float32), device="cuda")
    args = [M[k] for k in ("A", "B", "P", "Q", "m0", "S0")]
    full = ctx.lgssm_predict(y, *args, horizon=H, u=M["u"])
    tab = ctx.lgssm_predict(y, *args, horizon=H, u=M["u"], cov_shared_out=True)
    means_only = ctx.lgssm_predict(y, *args, horizon=H, u=M["u"], want_pred_cov=False, want_forecast_states=False)
    torch.cuda.synchronize()
    assert tab["pred_cov"].shape == (T + H, m, m) and tab["fc_cov"].shape == (H, d, d)
    assert torch.equal(full["pred_cov"], tab["pred_cov"][..., None].expand_as(full["pred_cov"]))
    assert torch.equal(full["fc_cov"], tab["fc_cov"][..., None].expand_as(full["fc_cov"]))
    assert torch.equal(full["pred_mean"], tab["pred_mean"]) and torch.equal(full["fc_mean"], tab["fc_mean"])
    assert means_only["pred_cov"] is None and means_only["fc_mean"] is None
    assert torch.equal(full["pred_mean"], means_only["pred_mean"])


# ---- port of test/inference/prediction_tests.jl:193-260 ("Predictions in State Space Models", tests #1 and #1.1): model_1
# is the LGSSM d = m = 1, A = B = P = Q = 1, x_0 ~ N(0, 1) one transition before x[1], with two forecast nodes o[1], o[2]
MISSING = None


@pytest.mark.parametrize("series", [[1.0, -500.0, MISSING, 100.0], [1.0, -500.0, MISSING, 100.0, MISSING, MISSING],
                                    [1.0, -500.0, 1.0, 100.0], [1.0, -500.0, 3.0, 100.0, 4.0, 5.0]])
def test_prediction_tests_model_1(rx, ctx, series):
    T, batch = len(series), 3
    one = np.ones((1, 1))
    model = rx.linear_gaussian_ssm_smoothing(one, one, one, one, (np.zeros(1), one), prior_on_previous_state=True, horizon=2)
    obs = np.array([0.0 if v is MISSING else v for v in series])
    mask = np.array([v is not MISSING for v in series], dtype=np.uint8)
    y = torch.tensor(np.repeat(obs[:, None, None], batch, axis=2), dtype=torch.float32, device="cuda")
    data = {"y": y}
    if not mask.all():
        data["ymask"] = torch.tensor(np.repeat(mask[:, None], batch, axis=1), device="cuda")
    res = rx.infer(model=model, data=data, predictvars={"o": rx.KeepLast()}, context=ctx)
    torch.cuda.synchronize()
    preds = res.predictions
    assert "o" in preds
    assert ("y" in preds) == (not mask.all())
    assert preds["o"].mean().shape[0] == 2
    if "y" in preds:
        assert preds["y"].mean().shape[0] == len(series)
    assert res.posteriors["x"].mean().shape[0] == T + 2
    ref = predict_reference_schedule(np.repeat(obs[:, None, None], batch, axis=2), one, one, one, one, np.zeros(1), one,
                                     np.repeat(mask[:, None], batch, axis=1), transition_first=True, horizon=2)
    assert rel_l2(preds["o"].mean().cpu().numpy(), ref["pred_mean"][T:]) < TOL_MEAN
    assert rel_l2(preds["o"].cov().cpu().numpy(), ref["pred_cov"][T:]) < TOL_COV
    if "y" in preds:
        assert rel_l2(preds["y"].mean().cpu().numpy(), ref["pred_mean"][:T]) < TOL_MEAN
        assert rel_l2(preds["y"].cov().cpu().numpy(), ref["pred_cov"][:T]) < TOL_COV
    # no predictvars: the call is the plain smoother, with no predictions
    plain = rx.infer(model=rx.linear_gaussian_ssm_smoothing(one, one, one, one, (np.zeros(1), one), prior_on_previous_state=True),
                     data=data, context=ctx)
    assert plain.predictions == {}


def test_conditioning_stress(ctx):
    """Observations dominate (Q = 1e-2 I, P = 1e2 I): D_t = Q - B S_s B' is a difference of nearly equal matrices."""
    d = m = 4
    T, batch, H = 200, 64, 3
    rng = np.random.default_rng(77)
    A = np.zeros((4, 4))
    c1, s1, c2, s2 = np.cos(np.pi / 15), np.sin(np.pi / 15), np.cos(np.pi / 35), np.sin(np.pi / 35)
    A[:2, :2] = [[c1, -s1], [s1, c1]]; A[2:, 2:] = [[c2, -s2], [s2, c2]]
    M = dict(A=A, B=np.diag([1.3, 0.7, 1.3, 0.7]), P=1e2 * np.eye(d), Q=1e-2 * np.eye(m), m0=np.zeros(d), S0=100.0 * np.eye(d))
    M = {k: v.astype(np.float32).astype(np.float64) for k, v in M.items()}
    y = (10.0 * rng.standard_normal((T, m, batch))).astype(np.float32)
    args = [M[k] for k in ("A", "B", "P", "Q", "m0", "S0")]
    ref = predict_reference_schedule(y, *args, horizon=H)
    # table route: S_s comes from the fp64 gain recursion (rounded once), so D_t keeps enough digits
    r = ctx.lgssm_predict(torch.tensor(y, device="cuda"), *args, horizon=H, want_status=True)
    torch.cuda.synchronize()
    em, ec = rel_l2(r["pred_mean"].cpu().numpy(), ref["pred_mean"]), rel_l2(r["pred_cov"].cpu().numpy(), ref["pred_cov"])
    # per-chain route: S_s is the fp32 output of the per-chain recursion; D_t = Q - B S_s B' (~1e-4 Q here) can lose every
    # digit, and a chain whose D_t is not SPD must be flagged, never returned silently
    rb = ctx.lgssm_predict(torch.tensor(y, device="cuda"), *args, horizon=H, force_per_chain_path=True, want_status=True)
    torch.cuda.synchronize()
    st = rb["status"].cpu().numpy()
    ok = st == 0
    emb = rel_l2(rb["pred_mean"].cpu().numpy()[..., ok], ref["pred_mean"][..., ok]) if ok.any() else float("nan")
    print(f"conditioning stress: table route rel. errors mean {em:.3e}, cov {ec:.3e}; per-chain route: "
          f"{int((~ok).sum())} of {batch} chains flagged NOT_SPD, mean error of the others {emb:.3e}")
    assert (r["status"].cpu().numpy() == 0).all()
    assert em < STRESS_TOL_MEAN and ec < TOL_COV
    assert set(np.unique(st)) <= {0, 4}
    assert not ok.any() or emb < STRESS_TOL_MEAN


def test_argument_errors(rx, ctx):
    L = rx._lib
    lib = L.load()
    d = m = 2
    T, batch = 4, 8
    host = [np.eye(2, dtype=np.float32) for _ in range(6)]
    hp = [h.ctypes.data_as(L.fp) for h in host]
    null_u8, null_i32, nf = ctypes.cast(None, L.u8p), ctypes.cast(None, L.i32p), L.as_fp(0)

    def call(y, mean, cov, pm, H, flags):
        return lib.rxg_lgssm_smooth_predict_f32(ctx.h, d, m, T, H, batch, *hp, nf, L.as_fp(y.data_ptr()), null_u8,
                                                L.as_fp(mean.data_ptr()), L.as_fp(cov.data_ptr()), nf,
                                                L.as_fp(pm.data_ptr()) if pm is not None else nf, nf, nf, nf, null_i32, flags)
    yc, mc, cc, pc = torch.zeros(T, m, batch), torch.zeros(T, d, batch), torch.zeros(T, d, d, batch), torch.zeros(T, m, batch)
    assert call(yc, mc, cc, pc, 0, 0) == L.RXG_ERR_UNSUPPORTED                    # host pointers
    yd, md, cd, pd = (t.cuda() for t in (yc, mc, cc, pc))
    assert call(yd, md, cd, pd, -1, L.PTR_DEVICE) == L.RXG_ERR_BAD_ARG            # H < 0
    assert call(yd, md, cd, None, 0, L.PTR_DEVICE) == L.RXG_ERR_BAD_ARG           # pred_mean == NULL
    assert call(yd, md, cd, pd, 0, L.PTR_DEVICE) == L.RXG_OK


@pytest.mark.parametrize("H", [0, 2])
def test_first_call_on_a_fresh_context_with_a_per_chain_model(rx, H):
    """A per-chain model with caller-owned forecast buffers needs no scratch: the first call on a new context must work."""
    fresh = rx.Context(0)
    try:
        d, m, T, batch = 4, 4, 20, 6
        rng = np.random.default_rng(31)
        M = _model(d, m, 41, batch)
        D = _dev_model(M)
        y = rng.standard_normal((T, m, batch)).astype(np.float32)
        r = fresh.lgssm_predict(torch.tensor(y, device="cuda"), *[D[k] for k in ("A", "B", "P", "Q", "m0", "S0")], horizon=H,
                                u=D["u"], per_chain_model=True, want_status=True)
        torch.cuda.synchronize()
        ref = predict_reference_schedule(y, M["A"], M["B"], M["P"], M["Q"], M["m0"], M["S0"], u=M["u"], horizon=H)
        _check(r, ref, H)
    finally:
        fresh.close()


@pytest.mark.parametrize("d,m,mask_kind", [(4, 4, "none"), (2, 1, "shared"), (6, 6, "none")])
def test_without_posterior_covariance_output(ctx, d, m, mask_kind):
    """post_cov = NULL at a register-resident shape: the family's own covariance table feeds the post-pass."""
    T, batch, H = 45, 33, 5
    M = _model(d, m, 51 + d)
    rng = np.random.default_rng(13)
    y = rng.standard_normal((T, m, batch)).astype(np.float32)
    mask = None
    if mask_kind == "shared":
        mask = np.ones(T, dtype=np.uint8); mask[[0, 9, T - 1]] = 0
    args = [M[k] for k in ("A", "B", "P", "Q", "m0", "S0")]
    yd = torch.tensor(y, device="cuda")
    r = ctx.lgssm_predict(yd, *args, horizon=H, u=M["u"], mask=mask, want_cov=False, want_status=True)
    full = ctx.lgssm_predict(yd, *args, horizon=H, u=M["u"], mask=mask)
    torch.cuda.synchronize()
    assert r["cov"] is None
    ref = predict_reference_schedule(y, *args, mask, u=M["u"], horizon=H)
    _check(r, ref, H)
    for k in ("mean", "pred_mean", "pred_cov", "fc_mean", "fc_cov"):
        assert torch.equal(r[k], full[k]), k


def test_without_posterior_covariance_output_unsupported_shape_runs_nothing(rx, ctx):
    M = _model(5, 3, 61)
    y = torch.zeros(10, 3, 8, device="cuda")
    before = ctx.launches
    with pytest.raises(rx.RxGaussError) as e:
        ctx.lgssm_predict(y, *[M[k] for k in ("A", "B", "P", "Q", "m0", "S0")], horizon=2, want_cov=False)
    assert e.value.code == rx._lib.RXG_ERR_UNSUPPORTED
    assert ctx.launches == before


def test_infer_raises_on_flagged_chains(rx, ctx):
    """Per-chain route in the observation-dominated regime (Q = 1e-2 I, P = 1e2 I, as test_conditioning_stress): infer raises
    exactly when a chain is flagged, and never returns a flagged chain's prediction."""
    d = m = 4
    T, batch = 200, 16
    rng = np.random.default_rng(77)
    A = np.zeros((4, 4))
    c1, s1, c2, s2 = np.cos(np.pi / 15), np.sin(np.pi / 15), np.cos(np.pi / 35), np.sin(np.pi / 35)
    A[:2, :2] = [[c1, -s1], [s1, c1]]; A[2:, 2:] = [[c2, -s2], [s2, c2]]
    model = rx.linear_gaussian_ssm_smoothing(A, np.diag([1.3, 0.7, 1.3, 0.7]), 1e2 * np.eye(d), 1e-2 * np.eye(m),
                                             (np.zeros(d), 100.0 * np.eye(d)))
    y = torch.tensor((10.0 * rng.standard_normal((T, m, batch))).astype(np.float32), device="cuda")
    mask = np.ones((T, batch), dtype=np.uint8); mask[5, 0] = 0
    md = torch.tensor(mask, device="cuda")
    st = ctx.lgssm_predict(y, model.A, model.B, model.P, model.Q, *model.x0, mask=md, want_status=True)["status"]
    torch.cuda.synchronize()
    flagged = bool((st != 0).any())
    print(f"observation-dominated per-chain route: {int((st != 0).sum())} of {batch} chains flagged")
    if flagged:
        with pytest.raises(rx.RxGaussError):
            rx.infer(model=model, data={"y": y, "ymask": md}, predictvars={"y": rx.KeepLast()}, context=ctx)
    else:
        res = rx.infer(model=model, data={"y": y, "ymask": md}, predictvars={"y": rx.KeepLast()}, context=ctx)
        assert bool(torch.isfinite(res.predictions["y"].mean()).all())
