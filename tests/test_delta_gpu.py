"""Delta node on the GPU: every chain of the NVRTC-compiled smoother and streaming filter against the fp64 oracle
(oracle/delta.py) for Linearization and Unscented, linear maps against the LGSSM smoother, chunked streams against one
call, the paper's pendulum experiment through infer(datastream=...), the module cache and the refusals.

Tolerances: the repository's (tests/util.py), relative L2 for means and relative Frobenius for covariances, checked
over all (t, k, chain) and for the means also on the worst chain."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import delta as D
from oracle import lgssm
from util import TOL_COV, TOL_MEAN, rel_l2

from delta_models import D8_F, D8_G, D8_SRC, PENDULUM_SRC, TRACKER_F, TRACKER_G, TRACKER_SRC, simulate

pytestmark = pytest.mark.gpu

LIN, UT = 0, 1
METHODS = {LIN: "linearization", UT: "unscented"}


def _dev(a, dtype=torch.float32):
    return torch.as_tensor(np.ascontiguousarray(a), dtype=dtype, device="cuda:0")


def _f32(*arrays):
    return [np.asarray(a, np.float32).astype(np.float64) for a in arrays]


def _compare(r, ref, method, what):
    tm, tc = TOL_MEAN, TOL_COV
    em = rel_l2(r["mean"].cpu().numpy(), ref["mean"])
    ec = rel_l2(r["cov"].cpu().numpy(), ref["cov"])
    # chain by chain: the worst chain, not only the aggregate
    mc = r["mean"].cpu().numpy()
    worst = max(rel_l2(mc[..., b], ref["mean"][..., b]) for b in range(mc.shape[-1]))
    print(f"{what} {METHODS[method]}: mean relL2 {em:.2e} (worst chain {worst:.2e}), cov relF {ec:.2e}")
    assert em < tm and worst < tm and ec < tc, (what, METHODS[method], em, worst, ec)
    assert int(r["status"].abs().sum()) == 0


def _pendulum_case(T, batch, seed, masked):
    P, Q = _f32(1e-4 * np.eye(2), [[0.05]])
    m0, S0 = _f32([0.5, 0.0], 0.01 * np.eye(2))
    B = np.array([[1.0, 0.0]])
    y = simulate(D.PENDULUM, None, B, P, Q, m0, S0, T, batch, seed).astype(np.float32)
    mask = None
    if masked:
        mask = (np.random.default_rng(seed + 1).random((T, batch)) > 0.2).astype(np.uint8)
        mask[:5] = 1
    return dict(P=P, Q=Q, m0=m0, S0=S0, B=B, y=y, mask=mask)


@pytest.mark.parametrize("method", [LIN, UT])
def test_pendulum_smoother_T1000_masked_every_chain(ctx, method):
    c = _pendulum_case(1000, 37, 11, masked=True)
    mod = ctx.delta_model(PENDULUM_SRC, "pendulum", 2, 1, method)
    r = ctx.delta_smooth(mod, _dev(c["y"]), c["m0"], c["S0"], c["P"], c["Q"], B=c["B"], mask=c["mask"],
                         want_filtered=True)
    ref = D.smooth(c["y"].astype(np.float64), D.PENDULUM, c["P"], c["m0"], c["S0"], METHODS[method], B=c["B"], Q=c["Q"],
                   mask=c["mask"])
    _compare(r, ref, method, "smoothed")
    _compare(dict(mean=r["filt_mean"], cov=r["filt_cov"], status=r["status"]),
             dict(mean=ref["filt_mean"], cov=ref["filt_cov"]), method, "filtered")


@pytest.mark.parametrize("method", [LIN, UT])
def test_range_bearing_tracker_every_chain(ctx, method):
    P, Q = _f32(np.diag([1e-3, 1e-3, 1e-2, 1e-2]), np.diag([0.01, 0.001]))
    m0, S0 = _f32([1.0, 2.0, 0.5, -0.3], np.diag([0.1, 0.1, 0.05, 0.05]))
    y = simulate(TRACKER_F, TRACKER_G, None, P, Q, m0, S0, 150, 45, 3).astype(np.float32)
    mod = ctx.delta_model(TRACKER_SRC, "cv", 4, 2, method, g_name="range_bearing")
    r = ctx.delta_smooth(mod, _dev(y), m0, S0, P, Q)
    ref = D.smooth(y.astype(np.float64), TRACKER_F, P, m0, S0, METHODS[method], g=TRACKER_G, Q=Q)
    _compare(r, ref, method, "tracker")


@pytest.mark.parametrize("method", [LIN, UT])
def test_d8_every_chain(ctx, method):
    P, Q = _f32(0.01 * np.eye(8), 0.1 * np.eye(3))
    m0, S0 = _f32(np.linspace(-1, 1, 8), 0.2 * np.eye(8))
    y = simulate(D8_F, D8_G, None, P, Q, m0, S0, 60, 33, 8).astype(np.float32)
    mask = (np.random.default_rng(9).random((60, 33)) > 0.3).astype(np.uint8)
    mod = ctx.delta_model(D8_SRC, "f8", 8, 3, method, g_name="g8")
    r = ctx.delta_smooth(mod, _dev(y), m0, S0, P, Q, mask=mask)
    ref = D.smooth(y.astype(np.float64), D8_F, P, m0, S0, METHODS[method], g=D8_G, Q=Q, mask=mask)
    _compare(r, ref, method, "d = 8")


LINEAR_SRC = """
template <class S> __device__ void lin_f(const S* x, S* z) {
    z[0] = 0.9 * x[0] + 0.2 * x[1]; z[1] = -0.1 * x[0] + 0.8 * x[1] + 0.1 * x[3];
    z[2] = 0.95 * x[2] + 0.05 * x[0]; z[3] = 0.7 * x[3] - 0.2 * x[2];
}
template <class S> __device__ void lin_g(const S* x, S* y) {
    y[0] = x[0] + 0.5 * x[2]; y[1] = x[1] - x[3];
}
"""
LIN_A = np.array([[0.9, 0.2, 0, 0], [-0.1, 0.8, 0, 0.1], [0.05, 0, 0.95, 0], [0, 0, -0.2, 0.7]])
LIN_B = np.array([[1.0, 0, 0.5, 0], [0, 1.0, 0, -1.0]])


@pytest.mark.parametrize("method", [LIN, UT])
@pytest.mark.parametrize("observe", ["B", "g"])
def test_linear_maps_match_the_lgssm_smoother(ctx, method, observe):
    mod = dict(A=LIN_A, B=LIN_B, P=0.1 * np.eye(4), Q=0.3 * np.eye(2), m0=np.array([1.0, -1, 0.5, 0]), S0=np.eye(4))
    mod = {k: np.asarray(v, np.float32).astype(np.float64) for k, v in mod.items()}
    _, y = lgssm.generate_data(mod, 200, 70, seed=21)
    yd = _dev(y)
    base = ctx.lgssm(yd, **mod, smooth=True)
    dm = ctx.delta_model(LINEAR_SRC, "lin_f", 4, 2, method, g_name="lin_g" if observe == "g" else None)
    r = ctx.delta_smooth(dm, yd, mod["m0"], mod["S0"], mod["P"], mod["Q"], B=mod["B"] if observe == "B" else None)
    e = [rel_l2(r["mean"].cpu().numpy(), base["mean"].cpu().numpy()), rel_l2(r["cov"].cpu().numpy(), base["cov"].cpu().numpy())]
    ref = lgssm.smooth_reference_schedule(y, **mod)
    e += [rel_l2(r["mean"].cpu().numpy(), ref["mean"]), rel_l2(r["cov"].cpu().numpy(), ref["cov"])]
    print(f"linear maps ({observe}) {METHODS[method]}: vs rxg_lgssm_smooth_f32 mean {e[0]:.2e} cov {e[1]:.2e}; "
          f"vs the fp64 LGSSM oracle mean {e[2]:.2e} cov {e[3]:.2e}")
    assert e[0] < TOL_MEAN and e[1] < TOL_COV and e[2] < TOL_MEAN and e[3] < TOL_COV, e


def _stream(ctx, mod, y, splits, gamma, mask=None):
    batch = y.shape[-1]
    d = mod.d
    cm = _dev(np.repeat(np.array([0.5, 0.0])[:, None], batch, 1))
    cc = _dev(np.repeat((0.01 * np.eye(2))[:, :, None], batch, 2))
    ct = _dev(np.repeat(np.array([[1.0], [0.01]]), batch, 1)) if gamma else None
    outs, t0 = [], 0
    for n in splits:
        kw = dict(B=np.array([[1.0, 0.0]]), carry_tau=ct, iters=5) if gamma else dict(B=np.array([[1.0, 0.0]]),
                                                                                        Q=np.array([[0.05]]))
        r = ctx.delta_filter_chunk(mod, y[t0:t0 + n].contiguous(), np.zeros((d, d)), cm, cc,
                                   mask=None if mask is None else mask[t0:t0 + n], **kw)
        assert int(r["status"].abs().sum()) == 0
        outs.append(r)
        t0 += n
    cat = {k: torch.cat([o[k] for o in outs]) for k in ("mean", "cov") + (("tau",) if gamma else ())}
    return cat, cm, cc, ct


@pytest.mark.parametrize("method", [LIN, UT])
@pytest.mark.parametrize("gamma", [False, True])
def test_chunk_splits_equal_one_call(ctx, method, gamma):
    _, _, obs = D.dataset(300, seed=5)
    y = _dev(np.repeat(obs[:, None, None], 40, 2) + np.random.default_rng(2).normal(0, 0.1, (300, 1, 40)))
    mask = _dev((np.random.default_rng(4).random((300, 40)) > 0.1), torch.uint8)
    mod = ctx.delta_model(PENDULUM_SRC, "pendulum", 2, 1, method)
    one = _stream(ctx, mod, y, [300], gamma, mask)
    split = _stream(ctx, mod, y, [1, 99, 37, 163], gamma, mask)
    for k in one[0]:
        assert torch.equal(one[0][k], split[0][k]), k
    for a, b in zip(one[1:], split[1:]):
        if a is not None:
            assert torch.equal(a, b)


@pytest.mark.parametrize("method", [LIN, UT])
def test_filter_with_known_noise_every_chain(ctx, method):
    c = _pendulum_case(400, 50, 17, masked=True)
    mod = ctx.delta_model(PENDULUM_SRC, "pendulum", 2, 1, method)
    cm = _dev(np.repeat(c["m0"][:, None], 50, 1))
    cc = _dev(np.repeat(c["S0"][:, :, None], 50, 2))
    r = ctx.delta_filter_chunk(mod, _dev(c["y"]), c["P"], cm, cc, Q=c["Q"], B=c["B"], mask=_dev(c["mask"], torch.uint8))
    fm, fc = np.zeros((400, 2, 50)), np.zeros((400, 2, 2, 50))
    for b in range(50):
        m_, c_ = D.filter_stream(c["y"][:, :, b].astype(np.float64), D.PENDULUM, c["P"], c["m0"], c["S0"],
                                 METHODS[method], B=c["B"], Q=c["Q"], mask=c["mask"][:, b])
        fm[..., b], fc[..., b] = m_, c_
    _compare(r, dict(mean=fm, cov=fc), method, "streaming filter")


@pytest.mark.parametrize("method", [LIN, UT])
def test_paper_pendulum_experiment_through_infer(ctx, method):
    """paper/example.jl: dataset(T = 1000, precision = 1.0) on chain 0 (seed 42), other seeds on the other chains;
    5 VMP iterations per datum, keephistory = 1000, chain by chain against the oracle."""
    from rxinfer_jl_b200 import inference as I
    T, batch = 1000, 19
    obs = np.stack([D.dataset(T, precision=1.0, seed=42 + b)[2] for b in range(batch)], axis=1)     # [T, batch]
    model = I.nonlinear_gamma_streaming(f=I.CudaFunction(PENDULUM_SRC, "pendulum", 2, 2), c=[1.0, 0.0])
    meta = {"f": I.Linearization() if method == LIN else I.Unscented()}
    chunks = [_dev(obs[i:i + 250]) for i in range(0, T, 250)]
    eng = I.infer(model=model, datastream=chunks, batch=batch, iterations=5, keephistory=T, constraints=I.MeanField(),
                  meta=meta, context=ctx)
    h = eng.history
    ini = D.PENDULUM_INIT
    worst = 0.0
    for b in range(batch):
        om, oc, oa, ob = D.vmp_gamma_stream(obs[:, b], D.PENDULUM, np.zeros((2, 2)), [1.0, 0.0], ini["mean"], ini["cov"],
                                            ini["shape"], 1.0 / ini["scale"], 5, METHODS[method])
        gm = h["state"].mu[..., b].cpu().numpy()
        gc = h["state"].Sigma[..., b].cpu().numpy()
        ga, gb = h["noise"].a[:, b].cpu().numpy(), h["noise"].b[:, b].cpu().numpy()
        e = max(rel_l2(gm, om), rel_l2(gc, oc), rel_l2(ga, oa), rel_l2(gb, ob))
        worst = max(worst, e)
    print(f"paper pendulum {METHODS[method]}: worst chain relL2 {worst:.2e}")
    assert worst < TOL_MEAN, worst
    assert eng.posteriors["noise"].a.shape == (batch,)


def test_unscented_parameters_reach_the_kernel(ctx):
    """Non-default (alpha, beta, kappa) against the oracle with the same parameters; with a wide prior and process noise
    the result differs from the defaults' by far more than the tolerance, so parameters lost on the way would fail."""
    ut = (0.5, 2.0, 1.0)
    P, Q = _f32(0.05 * np.eye(2), [[0.5]])
    m0, S0 = _f32([0.5, 0.0], 0.5 * np.eye(2))
    B = np.array([[1.0, 0.0]])
    y = simulate(D.PENDULUM, None, B, P, Q, m0, S0, 100, 45, 7).astype(np.float32)
    mod = ctx.delta_model(PENDULUM_SRC, "pendulum", 2, 1, UT, ut=ut)
    r = ctx.delta_smooth(mod, _dev(y), m0, S0, P, Q, B=B)
    ref = D.smooth(y.astype(np.float64), D.PENDULUM, P, m0, S0, "unscented", B=B, Q=Q, ut=ut)
    _compare(r, ref, UT, "unscented (0.5, 2, 1)")
    default = D.smooth(y.astype(np.float64), D.PENDULUM, P, m0, S0, "unscented", B=B, Q=Q)
    assert rel_l2(r["mean"].cpu().numpy(), default["mean"]) > 10 * TOL_MEAN


def test_streaming_refuses_a_wrongly_shaped_mask(ctx):
    from rxinfer_jl_b200 import inference as I
    model = I.nonlinear_gamma_streaming(f=I.CudaFunction(PENDULUM_SRC, "pendulum", 2, 2), c=[1.0, 0.0])
    eng = I.infer(model=model, datastream=None, autoupdates=True, batch=3, iterations=2, keephistory=10,
                  constraints=I.MeanField(), meta={"f": I.Linearization()}, context=ctx)
    before = eng.posteriors["state"].mu.clone()
    y = _dev(np.zeros((4, 3)))
    for bad in (np.ones(4, np.uint8), np.ones((3, 4), np.uint8)):     # one flag per step; transposed
        with pytest.raises(ValueError, match="mask must be"):
            eng.push({"y": y, "ymask": bad})
    assert torch.equal(eng.posteriors["state"].mu, before) and eng.ticks == 0
    eng.push({"y": y, "ymask": np.ones((4, 3), np.uint8)})
    assert eng.ticks == 4


def test_module_cache_compiles_once(ctx):
    src = PENDULUM_SRC + "\n// cache probe\n"
    n0 = ctx.delta_compiles
    a = ctx.delta_model(src, "pendulum", 2, 1, UT, ut=(0.1, 2.0, 0.0))
    n1 = ctx.delta_compiles
    b = ctx.delta_model(src, "pendulum", 2, 1, UT, ut=(0.1, 2.0, 0.0))
    assert n1 == n0 + 1 and ctx.delta_compiles == n1 and a.h.value == b.h.value
    ctx.delta_model(src, "pendulum", 2, 1, UT, ut=(0.2, 2.0, 0.0))      # other parameters: another module
    assert ctx.delta_compiles == n1 + 1


def test_refusals(ctx, rx):
    L = rx._lib
    lib = ctx.lib
    mod = ctx.delta_model(PENDULUM_SRC, "pendulum", 2, 1, LIN)
    with pytest.raises(rx.RxGaussError) as e:
        ctx.delta_model("template <class S> __device__ void f(const S* x, S* z) { z[0] = ; }", "f", 1, 1, LIN)
    assert e.value.code == L.RXG_ERR_BAD_ARG and "error" in str(e.value)
    with pytest.raises(rx.RxGaussError) as e:
        ctx.delta_model(PENDULUM_SRC, "pendulum", 9, 1, LIN)
    assert e.value.code == L.RXG_ERR_BAD_ARG
    y = _dev(np.zeros((4, 1, 3)))
    z = np.zeros(2, np.float32)
    E = np.eye(2, dtype=np.float32)
    one = np.ones((1, 1), np.float32)
    B = np.array([[1.0, 0.0]], np.float32)
    fp = lambda a: a.ctypes.data_as(L.fp)
    out = [_dev(np.zeros((4, 2, 3))), _dev(np.zeros((4, 2, 2, 3)))]
    args = (4, 3, fp(z), fp(E), fp(E), fp(B), fp(one), L.as_fp(y.data_ptr()), ctypes.cast(None, L.u8p),
            L.as_fp(out[0].data_ptr()), L.as_fp(out[1].data_ptr()), L.as_fp(0), L.as_fp(0), ctypes.cast(None, L.i32p))
    assert lib.rxg_delta_smooth_f32(None, mod.h, *args, L.PTR_DEVICE) == L.RXG_ERR_BAD_ARG          # null context
    assert lib.rxg_delta_smooth_f32(ctx.h, mod.h, *args, 0) == L.RXG_ERR_UNSUPPORTED                # host pointers
    assert lib.rxg_delta_smooth_f32(ctx.h, None, *args, L.PTR_DEVICE) == L.RXG_ERR_BAD_ARG          # no model
    bad = np.array([[-1.0]], np.float32)
    args_bad = args[:6] + (fp(bad),) + args[7:]
    assert lib.rxg_delta_smooth_f32(ctx.h, mod.h, *args_bad, L.PTR_DEVICE) == L.RXG_ERR_NOT_SPD     # Q not SPD
    assert lib.rxg_delta_smooth_f32(ctx.h, mod.h, *args, L.PTR_DEVICE) == L.RXG_OK
    cm, cc, ct = _dev(np.zeros((2, 3))), _dev(np.repeat(E[:, :, None], 3, 2)), _dev(np.ones((2, 3)))
    with pytest.raises(rx.RxGaussError) as e:           # a learned precision takes no Q
        ctx.delta_filter_chunk(mod, y, E, cm, cc, Q=one, B=B, carry_tau=ct, iters=2)
    assert e.value.code == L.RXG_ERR_BAD_ARG
    tr = ctx.delta_model(TRACKER_SRC, "cv", 4, 2, LIN, g_name="range_bearing")
    with pytest.raises(rx.RxGaussError) as e:           # ... and needs m = 1 and a linear row
        ctx.delta_filter_chunk(tr, _dev(np.zeros((4, 2, 3))), np.eye(4), _dev(np.zeros((4, 3))),
                               _dev(np.repeat(np.eye(4)[:, :, None], 3, 2)), carry_tau=ct, iters=2)
    assert e.value.code == L.RXG_ERR_BAD_ARG
    # a covariance that is not SPD is flagged per chain, not raised
    cc_bad = _dev(np.repeat(np.diag([1.0, -1.0])[:, :, None], 3, 2))
    r = ctx.delta_filter_chunk(ctx.delta_model(PENDULUM_SRC, "pendulum", 2, 1, UT), y, np.zeros((2, 2)), cm, cc_bad,
                               Q=one, B=B)
    assert (r["status"].cpu().numpy() == L.RXG_ERR_NOT_SPD).all()
