"""CPU checks of the observation predictions: the reference-schedule oracle against the closed form the kernels
evaluate, the forecast rows, the ``predictvars`` keyword handling of ``infer`` and the C entry's null-context check."""
import ctypes

import numpy as np
import pytest
import torch

from oracle.predict import predict_closed_form, predict_reference_schedule


def _random_model(rng, d, m):
    A = 0.9 * np.linalg.qr(rng.standard_normal((d, d)))[0]
    B = rng.standard_normal((m, d))
    G = rng.standard_normal((d, d)); P = G @ G.T / d + 0.1 * np.eye(d)
    G = rng.standard_normal((m, m)); Q = G @ G.T / m + 0.5 * np.eye(m)
    return A, B, P, Q, rng.standard_normal(d), 2.0 * np.eye(d)


def _rel(a, b):
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-300))


@pytest.mark.parametrize("d,m", [(1, 1), (4, 4), (4, 3), (3, 5)])
@pytest.mark.parametrize("H", [0, 3])
@pytest.mark.parametrize("transition_first", [False, True])
@pytest.mark.parametrize("with_u", [False, True])
def test_oracle_schedule_matches_closed_form(d, m, H, transition_first, with_u):
    rng = np.random.default_rng(100 * d + 10 * m + H)
    A, B, P, Q, m0, S0 = _random_model(rng, d, m)
    u = rng.standard_normal(d) if with_u else None
    T, batch = 11, 6
    y = rng.standard_normal((T, m, batch))
    mask = rng.random((T, batch)) > 0.3
    mask[-3:, 0] = False          # trailing gap
    mask[:, 1] = False            # prior-only chain
    mask[:, 2] = True
    r = predict_reference_schedule(y, A, B, P, Q, m0, S0, mask, u=u, transition_first=transition_first, horizon=H)
    c = predict_closed_form(y, A, B, P, Q, m0, S0, mask, u=u, transition_first=transition_first, horizon=H)
    assert r["pred_mean"].shape == (T + H, m, batch) and r["pred_cov"].shape == (T + H, m, m, batch)
    for k in ("pred_mean", "pred_cov", "mean", "cov"):
        assert _rel(r[k], c[k]) < 1e-10, k
    if H:
        for k in ("fc_mean", "fc_cov"):
            assert _rel(r[k], c[k]) < 1e-10, k


def test_oracle_forecast_rows_follow_the_recursion():
    rng = np.random.default_rng(7)
    d, m, T, H, batch = 3, 2, 8, 4, 3
    A, B, P, Q, m0, S0 = _random_model(rng, d, m)
    u = rng.standard_normal(d)
    y = rng.standard_normal((T, m, batch))
    r = predict_reference_schedule(y, A, B, P, Q, m0, S0, u=u, horizon=H)
    x, S = r["mean"][T - 1].T, np.transpose(r["cov"][T - 1], (2, 0, 1))
    for k in range(H):
        x = x @ A.T + u
        S = A @ S @ A.T + P
        np.testing.assert_allclose(r["fc_mean"][k].T, x, rtol=1e-10, atol=1e-10)
        np.testing.assert_allclose(np.transpose(r["fc_cov"][k], (2, 0, 1)), S, rtol=1e-10, atol=1e-10)
        np.testing.assert_allclose(r["pred_mean"][T + k].T, x @ B.T, rtol=1e-10, atol=1e-10)
        np.testing.assert_allclose(np.transpose(r["pred_cov"][T + k], (2, 0, 1)), B @ S @ B.T + Q, rtol=1e-10, atol=1e-10)


def _model(rx, horizon=0):
    return rx.linear_gaussian_ssm_smoothing(np.eye(2), np.eye(2), np.eye(2), np.eye(2), (np.zeros(2), np.eye(2)),
                                            horizon=horizon)


def test_infer_predictvars_keyword_handling(rx, monkeypatch):
    # every rejection happens before a context is created or a kernel launched
    from rxinfer_jl_b200 import inference

    def no_device(*a, **k):
        raise AssertionError("a device call was attempted")
    monkeypatch.setattr(inference, "default_context", no_device)
    y = torch.zeros(3, 2, 4)
    with pytest.raises(NotImplementedError):
        rx.infer(model=_model(rx), data={"y": y}, predictvars=rx.KeepEach())
    with pytest.raises(NotImplementedError):
        rx.infer(model=_model(rx), data={"y": y}, predictvars={"y": rx.KeepEach()})
    with pytest.raises(NotImplementedError):
        rx.infer(model=_model(rx, 2), data={"y": y}, predictvars={"z": rx.KeepLast()})
    with pytest.raises(NotImplementedError):
        rx.infer(model=_model(rx), data={"y": y}, predictvars=object())
    with pytest.raises(NotImplementedError):
        rx.infer(model=rx.hgf(), data={"y": y}, predictvars={"y": rx.KeepLast()})
    with pytest.raises(ValueError, match="horizon"):
        rx.infer(model=_model(rx), data={"y": y}, predictvars={"o": rx.KeepLast()})
    with pytest.raises(ValueError, match="`data` is not provided"):
        rx.infer(model=_model(rx), predictvars=rx.KeepLast(), batch=4)
    with pytest.raises(NotImplementedError, match="datastream"):
        rx.infer(model=_model(rx, 2), datastream=iter(()), batch=4)
    with pytest.raises(NotImplementedError, match="datastream"):
        rx.infer(model=_model(rx), datastream=iter(()), batch=4, predictvars={"y": rx.KeepLast()})
    assert rx.KeepLast() == rx.KeepLast() and rx.KeepLast() != rx.KeepEach()
    assert rx.InferenceResult(posteriors={}).predictions == {}


def test_predict_entry_refuses_a_null_context(rx):
    lib = rx._lib.load()
    null = ctypes.c_void_p(None)
    fpn = ctypes.cast(null, rx._lib.fp)
    rc = lib.rxg_lgssm_smooth_predict_f32(null, 4, 4, 1, 0, 1, fpn, fpn, fpn, fpn, fpn, fpn, fpn, fpn,
                                          ctypes.cast(null, rx._lib.u8p), fpn, fpn, fpn, fpn, fpn, fpn, fpn,
                                          ctypes.cast(null, rx._lib.i32p), rx._lib.PTR_DEVICE)
    assert rc == rx._lib.RXG_ERR_BAD_ARG
