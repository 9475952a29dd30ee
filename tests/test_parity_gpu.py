"""GPU parity tests for the fused LGSSM sweeps: CUDA path (through the C ABI) vs the fp64 oracle
on the same seeded inputs, against the committed golden fixtures, and -- at BASELINE.json's full
size -- through size-independent properties.  Tolerances are stated in tests/util.py."""
import os

import numpy as np
import pytest
import torch

from oracle import lgssm
from util import TOL_COV, TOL_MEAN, TOL_NLE, f32_model, rel_l2

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")


def dev(a, dtype=torch.float32):
    return torch.as_tensor(np.ascontiguousarray(a), dtype=dtype, device="cuda")


def check(r, ref, smooth=True, nle=True):
    km, kc = ("mean", "cov") if smooth else ("filt_mean", "filt_cov")
    assert rel_l2(r["mean"].cpu().numpy(), ref[km]) < TOL_MEAN
    if r["cov"] is not None:
        assert rel_l2(r["cov"].cpu().numpy(), ref[kc]) < TOL_COV
    if nle and r["neg_log_evidence"] is not None:
        g = r["neg_log_evidence"].cpu().numpy().astype(np.float64)
        den = np.maximum(np.abs(ref["neg_log_evidence"]), 1e-3)        # a chain without any datum has evidence 0
        assert np.max(np.abs(g - ref["neg_log_evidence"]) / den) < TOL_NLE


@pytest.mark.parametrize("d,T,batch", [(4, 64, 8), (2, 48, 6)])
def test_golden_fixture(ctx, d, T, batch):
    z = np.load(os.path.join(GOLD, f"lgssm_d{d}_T{T}_b{batch}.npz"))
    mod = {k[6:]: z[k] for k in z.files if k.startswith("model_")}
    ref = {k: z[k] for k in ("mean", "cov", "filt_mean", "filt_cov", "neg_log_evidence")}
    y = dev(z["y"])
    for force in (False, True):
        r = ctx.lgssm(y, **_kw(mod), smooth=True, want_evidence=True, want_status=True, force_per_chain_path=force)
        check(r, ref)
        assert int(r["status"].abs().sum()) == 0
        f = ctx.lgssm(y, **_kw(mod), smooth=False, want_evidence=True, force_per_chain_path=force)
        check(f, ref, smooth=False)


def _kw(mod):
    return dict(A=mod["A"], B=mod["B"], P=mod["P"], Q=mod["Q"], m0=mod["m0"], S0=mod["S0"])


@pytest.mark.parametrize("d", [2, 4])
@pytest.mark.parametrize("force", [False, True])
def test_smoothing_T1000_vs_oracle(ctx, d, force):
    """configs[0] shape (d, T = 1000) on a small batch the oracle finishes in seconds."""
    mod = f32_model(lgssm.notebook_model(d))
    _, y = lgssm.generate_data(mod, 1000, 96, seed=42)
    ref = lgssm.smooth_reference_schedule(y, **mod)
    r = ctx.lgssm(dev(y), **_kw(mod), smooth=True, want_evidence=True, want_status=True, force_per_chain_path=force)
    check(r, ref)
    assert int(r["status"].abs().sum()) == 0
    # covariances SPD (mlgssm_test.jl:126)
    cov = r["cov"].permute(0, 3, 1, 2).reshape(-1, d, d).double().cpu().numpy()
    assert bool((np.linalg.eigvalsh(cov) > 0).all())


def test_chains_per_thread_2_path(ctx, monkeypatch):
    mod = f32_model(lgssm.notebook_model(4))
    _, y = lgssm.generate_data(mod, 200, 64, seed=7)
    ref = lgssm.smooth_reference_schedule(y, **mod)
    for cpt in ("2", "1"):
        ctx.set_option("force_cpt", int(cpt))
        check(ctx.lgssm(dev(y), **_kw(mod), smooth=True, want_evidence=True), ref)
        check(ctx.lgssm(dev(y), **_kw(mod), smooth=True), ref, nle=False)
        check(ctx.lgssm(dev(y), **_kw(mod), smooth=False, want_evidence=True), ref, smooth=False)
    # ragged: batch not a multiple of 32 * CPT
    ctx.set_option("force_cpt", 2)
    _, y2 = lgssm.generate_data(mod, 90, 100, seed=8)
    check(ctx.lgssm(dev(y2), **_kw(mod), smooth=True, want_evidence=True), lgssm.smooth_reference_schedule(y2, **mod))


@pytest.mark.parametrize("d,m", [(1, 1), (2, 1), (3, 3), (4, 1), (4, 2), (6, 6)])
@pytest.mark.parametrize("force", [False, True])
def test_other_shapes(ctx, d, m, force):
    rng = np.random.default_rng(d * 10 + m)
    Aq, _ = np.linalg.qr(rng.standard_normal((d, d)))
    mod = f32_model(dict(A=0.95 * Aq, B=rng.standard_normal((m, d)), P=0.1 * np.eye(d), Q=2.0 * np.eye(m),
                         m0=rng.standard_normal(d), S0=10.0 * np.eye(d)))
    _, y = lgssm.generate_data(mod, 150, 40, seed=3)
    ref = lgssm.smooth_reference_schedule(y, **mod)
    r = ctx.lgssm(dev(y), **_kw(mod), smooth=True, want_evidence=True, force_per_chain_path=force)
    check(r, ref)


def test_edge_T1_and_prior_only(ctx):
    mod = f32_model(lgssm.notebook_model(4))
    _, y = lgssm.generate_data(mod, 1, 5, seed=1)
    ref = lgssm.smooth_reference_schedule(y, **mod)
    for force in (False, True):
        check(ctx.lgssm(dev(y), **_kw(mod), smooth=True, want_evidence=True, force_per_chain_path=force), ref)
    # T = 2 exercises exactly one backward step
    _, y2 = lgssm.generate_data(mod, 2, 5, seed=2)
    ref2 = lgssm.smooth_reference_schedule(y2, **mod)
    for force in (False, True):
        check(ctx.lgssm(dev(y2), **_kw(mod), smooth=True, want_evidence=True, force_per_chain_path=force), ref2)
    # all data missing => posterior == prior pushed through the dynamics
    mask = np.zeros((2, 5), dtype=np.uint8)
    refm = lgssm.smooth_reference_schedule(y2, **mod, mask=mask)
    rm = ctx.lgssm(dev(y2), **_kw(mod), smooth=True, mask=dev(mask, torch.uint8))
    assert rel_l2(rm["cov"].cpu().numpy(), refm["cov"]) < TOL_COV
    assert np.abs(rm["mean"].cpu().numpy() - refm["mean"]).max() < 1e-6


def test_ragged_batch_and_missing_data(ctx):
    mod = f32_model(lgssm.notebook_model(4))
    T, batch = 120, 77                                  # not a multiple of the block size
    _, y = lgssm.generate_data(mod, T, batch, seed=11)
    rng = np.random.default_rng(5)
    mask = (rng.random((T, batch)) > 0.25).astype(np.uint8)
    mask[-5:, 3] = 0
    ref = lgssm.smooth_reference_schedule(y, **mod, mask=mask)
    r = ctx.lgssm(dev(y), **_kw(mod), smooth=True, mask=dev(mask, torch.uint8), want_evidence=True, want_status=True)
    check(r, ref)
    r0 = ctx.lgssm(dev(y), **_kw(mod), smooth=True)
    check(r0, lgssm.smooth_reference_schedule(y, **mod), nle=False)


def test_per_chain_models(ctx):
    base = f32_model(lgssm.notebook_model(4))
    batch, T = 48, 100
    rng = np.random.default_rng(9)
    scale = 1.0 + rng.random(batch)
    mods = {k: np.stack([v * (scale[i] if k in ("P", "Q", "S0") else 1.0) for i in range(batch)]) for k, v in base.items()}
    mods = {k: v.astype(np.float32).astype(np.float64) for k, v in mods.items()}
    _, y = lgssm.generate_data(base, T, batch, seed=13)
    ref = lgssm.smooth_reference_schedule(y, **mods)
    # ABI layout: [r][c][batch]
    to_abi = lambda M: dev(np.moveaxis(M, 0, -1))
    r = ctx.lgssm(dev(y), A=to_abi(mods["A"]), B=to_abi(mods["B"]), P=to_abi(mods["P"]), Q=to_abi(mods["Q"]),
                  m0=to_abi(mods["m0"]), S0=to_abi(mods["S0"]), smooth=True, want_evidence=True,
                  per_chain_model=True)
    check(r, ref)


def test_streaming_filter_transition_first(ctx):
    mod = f32_model(lgssm.notebook_model(2))
    _, y = lgssm.generate_data(mod, 300, 33, seed=17)
    ref = lgssm.filter_streaming(y, **mod)
    for force in (False, True):
        r = ctx.lgssm(dev(y), **_kw(mod), smooth=False, transition_first=True, force_per_chain_path=force)
        assert rel_l2(r["mean"].cpu().numpy(), ref["mean"]) < TOL_MEAN
        assert rel_l2(r["cov"].cpu().numpy(), ref["cov"]) < TOL_COV


def test_cov_shared_out_and_host_pointer_path(ctx):
    mod = f32_model(lgssm.notebook_model(4))
    _, y = lgssm.generate_data(mod, 80, 24, seed=19)
    ref = lgssm.smooth_reference_schedule(y, **mod)
    r = ctx.lgssm(dev(y), **_kw(mod), smooth=True, cov_shared_out=True)
    assert tuple(r["cov"].shape) == (80, 4, 4)
    assert rel_l2(r["cov"].cpu().numpy(), ref["cov"][..., 0]) < TOL_COV
    assert rel_l2(r["mean"].cpu().numpy(), ref["mean"]) < TOL_MEAN
    # host pointers (pinned) staged by the library
    yh = torch.from_numpy(y).pin_memory()
    rh = ctx.lgssm(yh, **_kw(mod), smooth=True, want_evidence=True, want_status=True)
    assert not rh["mean"].is_cuda
    check(rh, ref)


def test_infer_entry_point(rx, ctx):
    mod = f32_model(lgssm.notebook_model(4))
    _, y = lgssm.generate_data(mod, 60, 16, seed=23)
    ref = lgssm.smooth_reference_schedule(y, **mod)
    res = rx.infer(model=rx.linear_gaussian_ssm_smoothing(mod["A"], mod["B"], mod["P"], mod["Q"], (mod["m0"], mod["S0"])),
                   data={"y": dev(y)}, free_energy=True, options={"limit_stack_depth": 500}, context=ctx)
    q = res.posteriors["x"]
    assert rel_l2(q.mean().cpu().numpy(), ref["mean"]) < TOL_MEAN
    assert rel_l2(q.cov().cpu().numpy(), ref["cov"]) < TOL_COV
    assert rel_l2(res.free_energy.cpu().numpy(), ref["neg_log_evidence"]) < TOL_NLE
    fil = rx.infer(model=rx.linear_gaussian_ssm_filtering(mod["A"], mod["B"], mod["P"], mod["Q"], (mod["m0"], mod["S0"])),
                   data={"y": dev(y)}, context=ctx)
    refs = lgssm.filter_streaming(y, **mod)
    assert rel_l2(fil.history["x_t"].mean().cpu().numpy(), refs["mean"]) < TOL_MEAN


def test_unsupported_shape_errors_loudly(rx, ctx):
    mod = lgssm.dense_model(65)
    y = torch.zeros(4, 65, 2, device="cuda")
    with pytest.raises(rx.RxGaussError) as e:
        ctx.lgssm(y, **_kw(mod), smooth=True)
    assert e.value.code == rx._lib.RXG_ERR_UNSUPPORTED


def test_full_size_properties(ctx, monkeypatch):
    """BASELINE.json configs[1] (d = 4, T = 1000, batch = 65 536): size-independent properties.
    (1) chains are independent: a slice re-run alone is bit-identical; (2) linearity of the
    posterior mean in (y, m0); (3) two chains fed the same series agree bit-exactly; (4) a sample
    of chains matches the oracle within the parity tolerance; (5) covariances SPD and identical
    across chains (shared model)."""
    mod = f32_model(lgssm.notebook_model(4))
    T, batch = 1000, 65536
    g = torch.Generator(device="cuda").manual_seed(1234)
    y = torch.randn(T, 4, batch, device="cuda", generator=g) * 3.0
    y[:, :, 1] = y[:, :, 0]
    r = ctx.lgssm(y, **_kw(mod), smooth=True, want_evidence=True)
    mean, cov = r["mean"], r["cov"]
    assert torch.equal(mean[:, :, 0], mean[:, :, 1])                                   # (3)
    ctx.set_option("force_cpt", 2)     # same kernel variant as the full batch (2 chains / thread, checkpoint mode)
    sub = ctx.lgssm(y[:, :, 4096:4096 + 512].contiguous(), **_kw(mod), smooth=True, want_evidence=True)
    ctx.set_option("force_cpt", 0)
    assert torch.equal(sub["mean"], mean[:, :, 4096:4096 + 512])                       # (1)
    r2 = ctx.lgssm((2.0 * y).contiguous(), A=mod["A"], B=mod["B"], P=mod["P"], Q=mod["Q"], m0=2.0 * mod["m0"],
                   S0=mod["S0"], smooth=True)
    assert rel_l2(r2["mean"][:, :, :2048].cpu().numpy(), 2.0 * mean[:, :, :2048].cpu().numpy()) < 1e-6   # (2)
    idx = [0, 777, 65535]
    ref = lgssm.smooth_reference_schedule(y[:, :, idx].cpu().numpy(), **mod)
    assert rel_l2(mean[:, :, idx].cpu().numpy(), ref["mean"]) < TOL_MEAN                # (4)
    assert rel_l2(cov[:, :, :, idx].cpu().numpy(), ref["cov"]) < TOL_COV
    nle = r["neg_log_evidence"][idx].cpu().numpy().astype(np.float64)
    assert np.max(np.abs(nle - ref["neg_log_evidence"]) / np.abs(ref["neg_log_evidence"])) < TOL_NLE
    assert torch.equal(cov[..., 0], cov[..., 65535])                                    # (5)
    assert bool((torch.linalg.eigvalsh(cov[..., 0].double()) > 0).all())
    # the per-chain path at full size agrees with the gain-table path
    rp = ctx.lgssm(y, **_kw(mod), smooth=True, force_per_chain_path=True)
    assert rel_l2(rp["mean"][:, :, ::97].cpu().numpy(), mean[:, :, ::97].cpu().numpy()) < 2 * TOL_MEAN


@pytest.mark.parametrize("T", [1, 2, 3, 1000, 1024, 1025, 2500, 5000])
def test_time_parallel_gain_scan_vs_sequential_and_oracle(ctx, monkeypatch, T):
    """The gain tables come from associative scans over time (rxg_gain.cuh).  They must agree with
    the sequential Riccati kernels (RXG_GAIN_SEQ=1) and with the fp64 oracle, including T > 1024
    where every scan thread owns several time steps."""
    mod = f32_model(lgssm.notebook_model(4))
    batch = 8
    _, y = lgssm.generate_data(mod, T, batch, seed=29)
    yd = dev(y)
    ctx.set_option("gain_seq", 0)
    a = ctx.lgssm(yd, **_kw(mod), smooth=True, want_evidence=True)
    f = ctx.lgssm(yd, **_kw(mod), smooth=False, transition_first=True)
    ctx.set_option("gain_seq", 1)
    b = ctx.lgssm(yd, **_kw(mod), smooth=True, want_evidence=True)
    fb = ctx.lgssm(yd, **_kw(mod), smooth=False, transition_first=True)
    assert rel_l2(a["cov"].cpu().numpy(), b["cov"].cpu().numpy()) < 1e-6
    assert rel_l2(a["mean"].cpu().numpy(), b["mean"].cpu().numpy()) < 1e-6
    assert rel_l2(f["cov"].cpu().numpy(), fb["cov"].cpu().numpy()) < 1e-6
    assert rel_l2(f["mean"].cpu().numpy(), fb["mean"].cpu().numpy()) < 1e-6
    if T <= 2500:
        ref = lgssm.smooth_reference_schedule(y, **mod)
        check(a, ref)


def test_gain_scan_other_shapes(ctx, monkeypatch):
    ctx.set_option("gain_seq", 0)
    for d, m in [(1, 1), (2, 1), (3, 3), (4, 2), (6, 6)]:
        rng = np.random.default_rng(100 + d * 10 + m)
        Aq, _ = np.linalg.qr(rng.standard_normal((d, d)))
        mod = f32_model(dict(A=0.9 * Aq, B=rng.standard_normal((m, d)), P=0.2 * np.eye(d), Q=1.5 * np.eye(m),
                             m0=rng.standard_normal(d), S0=5.0 * np.eye(d)))
        _, y = lgssm.generate_data(mod, 1300, 6, seed=31)
        check(ctx.lgssm(dev(y), **_kw(mod), smooth=True, want_evidence=True), lgssm.smooth_reference_schedule(y, **mod))


def test_host_pointer_path_sliced_pipeline(ctx, monkeypatch):
    """Host-pointer calls are cut into batch slices pipelined over three streams (H2D | sweep | D2H);
    force several slices on a ragged batch, with mask, evidence and status outputs."""
    mod = f32_model(lgssm.notebook_model(4))
    T, batch = 70, 203
    _, y = lgssm.generate_data(mod, T, batch, seed=37)
    rng = np.random.default_rng(11)
    mask = (rng.random((T, batch)) > 0.2).astype(np.uint8)
    yh = torch.from_numpy(y).pin_memory()
    for ns in ("5", "1"):
        ctx.set_option("host_slices", int(ns))
        r = ctx.lgssm(yh, **_kw(mod), smooth=True, want_evidence=True, want_status=True)
        check(r, lgssm.smooth_reference_schedule(y, **mod))
        assert int(r["status"].abs().sum()) == 0
        rm = ctx.lgssm(yh, **_kw(mod), smooth=True, mask=torch.from_numpy(mask).pin_memory(), want_evidence=True)
        check(rm, lgssm.smooth_reference_schedule(y, **mod, mask=mask))
        f = ctx.lgssm(yh, **_kw(mod), smooth=False, want_evidence=True)
        check(f, lgssm.smooth_reference_schedule(y, **mod), smooth=False)
    # pageable (unpinned) host memory is legal too, just slower
    rp = ctx.lgssm(torch.from_numpy(y.copy()), **_kw(mod), smooth=True)
    check(rp, lgssm.smooth_reference_schedule(y, **mod), nle=False)


@pytest.mark.parametrize("d,T,batch", [(4, 90, 203), (16, 40, 70)])
def test_host_pointer_covariance_broadcast_is_bit_identical(ctx, monkeypatch, d, T, batch):
    """Host-pointer calls of a shared model fetch the chain-independent covariance table once and broadcast it
    into the caller's per-chain buffer with host threads; the buffer must hold exactly the bits the full
    device->host copy (RXG_HOST_COV_D2H=1) delivers, for smoothing and filtering, sliced or not."""
    mod = f32_model(lgssm.notebook_model(d) if d <= 4 else lgssm.dense_model(d))
    _, y = lgssm.generate_data(mod, T, batch, seed=38)
    yh = torch.from_numpy(y).pin_memory()
    ctx.set_option("host_bcast_min_mb", 0)
    ctx.set_option("host_threads", 7)
    for smooth in (True, False):
        for ns in ("3", "1"):
            ctx.set_option("host_slices", int(ns))
            ctx.set_option("host_cov_d2h", 1)
            a = ctx.lgssm(yh, **_kw(mod), smooth=smooth, transition_first=not smooth)
            ctx.set_option("host_cov_d2h", 0)
            b = ctx.lgssm(yh, **_kw(mod), smooth=smooth, transition_first=not smooth)
            assert torch.equal(a["cov"], b["cov"]) and torch.equal(a["mean"], b["mean"])
    ref = lgssm.smooth_reference_schedule(y, **mod)
    r = ctx.lgssm(yh, **_kw(mod), smooth=True)
    assert rel_l2(r["cov"].numpy(), ref["cov"]) < TOL_COV and rel_l2(r["mean"].numpy(), ref["mean"]) < TOL_MEAN


@pytest.mark.parametrize("tf", [False, True])
def test_transition_offset_and_prior_on_previous_state(ctx, tf):
    """Fused `+` rule (constant offset u) and RXG_TRANSITION_FIRST, smoothing and filtering, both
    kernel families, plus per-chain offsets."""
    rng = np.random.default_rng(77)
    mod = f32_model(lgssm.notebook_model(4))
    u = rng.standard_normal(4).astype(np.float32).astype(np.float64)
    T, batch = 160, 50
    _, y = lgssm.generate_data(mod, T, batch, seed=41)
    y = (y + 2.0).astype(np.float32)
    ref = lgssm.smooth_reference_schedule(y, **mod, u=u, transition_first=tf)
    for force in (False, True):
        r = ctx.lgssm(dev(y), **_kw(mod), u=u, smooth=True, want_evidence=True, transition_first=tf, force_per_chain_path=force)
        check(r, ref)
        f = ctx.lgssm(dev(y), **_kw(mod), u=u, smooth=False, want_evidence=True, transition_first=tf, force_per_chain_path=force)
        check(f, ref, smooth=False)
    # per-chain model with per-chain offsets
    us = rng.standard_normal((batch, 4)).astype(np.float32).astype(np.float64)
    mods = {k: np.broadcast_to(v, (batch,) + v.shape).copy() for k, v in mod.items()}
    refp = lgssm.smooth_reference_schedule(y, **mods, u=us, transition_first=tf)
    to_abi = lambda M: dev(np.moveaxis(M, 0, -1))
    rp = ctx.lgssm(dev(y), A=to_abi(mods["A"]), B=to_abi(mods["B"]), P=to_abi(mods["P"]), Q=to_abi(mods["Q"]),
                   m0=to_abi(mods["m0"]), S0=to_abi(mods["S0"]), u=to_abi(us), smooth=True, want_evidence=True,
                   per_chain_model=True, transition_first=tf)
    check(rp, refp)


@pytest.mark.parametrize("d,T,batch", [(8, 120, 37), (16, 200, 70), (32, 150, 64), (64, 300, 96)])
def test_large_state_family(ctx, d, T, batch):
    """BASELINE configs[2] family (d = 64 and the smaller block sizes): dense A = 0.99 * Orth, B = I,
    shared model, gain tables from block-cooperative fp64 kernels, tiled mean sweep."""
    mod = f32_model(lgssm.dense_model(d, seed=64))
    _, y = lgssm.generate_data(mod, T, batch, seed=43)
    ref = lgssm.smooth_reference_schedule(y, **mod)
    r = ctx.lgssm(dev(y), **_kw(mod), smooth=True, want_status=True)
    check(r, ref, nle=False)
    assert int(r["status"].abs().sum()) == 0
    rs = ctx.lgssm(dev(y), **_kw(mod), smooth=True, cov_shared_out=True)
    assert tuple(rs["cov"].shape) == (T, d, d)
    assert rel_l2(rs["cov"].cpu().numpy(), ref["cov"][..., 0]) < TOL_COV
    f = ctx.lgssm(dev(y), **_kw(mod), smooth=False, transition_first=True)
    reff = lgssm.filter_streaming(y, **mod)
    assert rel_l2(f["mean"].cpu().numpy(), reff["mean"]) < TOL_MEAN
    assert rel_l2(f["cov"].cpu().numpy(), reff["cov"]) < TOL_COV


def _random_model(rng, d, m, scale_a=0.9):
    Aq, _ = np.linalg.qr(rng.standard_normal((d, d)))
    L = rng.standard_normal((d, d)) * 0.1
    return f32_model(dict(A=scale_a * Aq, B=rng.standard_normal((m, d)) / np.sqrt(d), P=0.2 * np.eye(d) + L @ L.T,
                          Q=1.5 * np.eye(m), m0=rng.standard_normal(d), S0=5.0 * np.eye(d)))


@pytest.mark.parametrize("d,m", [(5, 5), (5, 3), (7, 7), (3, 2), (2, 3), (6, 4), (10, 10), (12, 7), (24, 24), (33, 20), (64, 32)])
def test_general_shapes_shared_model(ctx, d, m):
    """Any (d, m) <= 64: shapes without a dedicated kernel family are embedded in the next native one (decoupled
    dummy coordinates; the evidence is corrected for the dummy observations).  Smoothing, filtering, evidence,
    transition offset, prior one transition earlier, de-duplicated covariance output."""
    rng = np.random.default_rng(1000 + 64 * d + m)
    mod = _random_model(rng, d, m)
    T, batch = 40, 37
    _, y = lgssm.generate_data(mod, T, batch, seed=d * 100 + m)
    u = (0.2 * rng.standard_normal(d)).astype(np.float32)
    for kw in (dict(), dict(u=u, transition_first=True)):
        kw64 = {k: (v.astype(np.float64) if k == "u" else v) for k, v in kw.items()}
        ref = lgssm.smooth_reference_schedule(y, **mod, **kw64)
        check(ctx.lgssm(dev(y), **_kw(mod), smooth=True, want_evidence=True, **kw), ref)
        check(ctx.lgssm(dev(y), **_kw(mod), smooth=False, want_evidence=True, **kw), ref, smooth=False)
    r = ctx.lgssm(dev(y), **_kw(mod), smooth=True, cov_shared_out=True)
    assert r["cov"].shape == (T, d, d)
    assert rel_l2(r["cov"].cpu().numpy(), ref0 := lgssm.smooth_reference_schedule(y, **mod)["cov"][..., 0]) < TOL_COV


@pytest.mark.parametrize("d,m", [(5, 3), (8, 8), (9, 4), (16, 16), (20, 12), (64, 64)])
def test_general_shapes_per_chain_and_masks(ctx, d, m):
    """Per-chain models, missing data and the forced per-chain path for shapes beyond the register kernels:
    lgssm_generic_chain_kernel (one CTA per chain, runtime d and m) -- round 1 returned RXG_ERR_UNSUPPORTED for d >= 8."""
    rng = np.random.default_rng(2000 + 64 * d + m)
    mod = _random_model(rng, d, m)
    T, batch = (24, 9) if d < 64 else (12, 5)
    _, y = lgssm.generate_data(mod, T, batch, seed=d + m)
    mask = (rng.random((T, batch)) > 0.3).astype(np.uint8)
    mask[-3:, 0] = 0                                         # trailing gap
    mask[:, 1] = 0                                           # prior only
    u = (0.2 * rng.standard_normal(d)).astype(np.float32)
    ref = lgssm.smooth_reference_schedule(y, **mod, mask=mask)
    r = ctx.lgssm(dev(y), **_kw(mod), smooth=True, mask=dev(mask, torch.uint8), want_evidence=True, want_status=True)
    check(r, ref)
    assert int(r["status"].abs().sum()) == 0
    f = ctx.lgssm(dev(y), **_kw(mod), smooth=False, mask=dev(mask, torch.uint8), want_evidence=True)
    check(f, ref, smooth=False)
    refu = lgssm.smooth_reference_schedule(y, **mod, u=u.astype(np.float64), transition_first=True)
    check(ctx.lgssm(dev(y), **_kw(mod), u=u, smooth=True, transition_first=True, force_per_chain_path=True, want_evidence=True), refu)
    # per-chain models: every chain its own (A, B, P, Q, m0, S0)
    mods = [_random_model(rng, d, m) for _ in range(batch)]
    stack = lambda k: dev(np.stack([mm[k] for mm in mods], axis=-1))
    rp = ctx.lgssm(dev(y), stack("A"), stack("B"), stack("P"), stack("Q"), stack("m0"), stack("S0"), smooth=True,
                   per_chain_model=True, want_evidence=True)
    for b in range(batch):
        rb = lgssm.smooth_reference_schedule(y[:, :, b:b + 1], **mods[b])
        assert rel_l2(rp["mean"][:, :, b].cpu().numpy(), rb["mean"][:, :, 0]) < 3 * TOL_MEAN
        assert rel_l2(rp["cov"][..., b].cpu().numpy(), rb["cov"][..., 0]) < TOL_COV
        assert abs(float(rp["neg_log_evidence"][b]) - rb["neg_log_evidence"][0]) / abs(rb["neg_log_evidence"][0]) < 5 * TOL_NLE


def test_large_state_offset_by_linearity(ctx):
    """Transition offset on the tensor-core family (round 1: RXG_ERR_UNSUPPORTED): removed by linearity, the sweep
    itself runs offset free; also through the streaming chunk entry."""
    rng = np.random.default_rng(9)
    mod = f32_model(lgssm.dense_model(16))
    u = (0.3 * rng.standard_normal(16)).astype(np.float32)
    _, y = lgssm.generate_data(mod, 50, 70, seed=12)
    for tf in (False, True):
        ref = lgssm.smooth_reference_schedule(y, **mod, u=u.astype(np.float64), transition_first=tf)
        check(ctx.lgssm(dev(y), **_kw(mod), u=u, smooth=True, transition_first=tf, want_evidence=True), ref)
        check(ctx.lgssm(dev(y), **_kw(mod), u=u, smooth=False, transition_first=tf, want_evidence=True), ref, smooth=False)


@pytest.mark.parametrize("d,T", [(16, 1), (16, 2), (16, 37), (32, 130), (64, 257)])
def test_large_state_doubling_vs_sequential(ctx, monkeypatch, d, T):
    """Large-state gain tables: forward by doubling + backward suffix scan (default) must agree with the
    sequential Riccati kernels (RXG_LARGE_SEQ=1) and the oracle, including T = 1, 2 and non powers of two."""
    mod = f32_model(lgssm.dense_model(d, seed=11))
    _, y = lgssm.generate_data(mod, T, 8, seed=47)
    yd = dev(y)
    ctx.set_option("large_seq", 0)
    a = ctx.lgssm(yd, **_kw(mod), smooth=True)
    fa = ctx.lgssm(yd, **_kw(mod), smooth=False, transition_first=True)
    ctx.set_option("large_seq", 1)
    b = ctx.lgssm(yd, **_kw(mod), smooth=True)
    fb = ctx.lgssm(yd, **_kw(mod), smooth=False, transition_first=True)
    for k in ("mean", "cov"):
        assert rel_l2(a[k].cpu().numpy(), b[k].cpu().numpy()) < 2e-6
        assert rel_l2(fa[k].cpu().numpy(), fb[k].cpu().numpy()) < 2e-6
    check(a, lgssm.smooth_reference_schedule(y, **mod), nle=False)


@pytest.mark.parametrize("d,T,batch", [(16, 90, 300), (32, 70, 129), (64, 50, 257)])
def test_large_state_tensor_core_vs_fp32_pipe(ctx, monkeypatch, d, T, batch):
    """d >= 16: the mean recursions run on the tensor cores (wgmma; u_t = K_t y_t pre-pass + [F;E] / G recursion, 3xTF32);
    RXG_NO_UMMA=1 runs the same tables through the FP32-pipe block sweep.  Ragged last chain tile, several
    time slices in the pre-pass; smoothing and filtering; both against each other and the oracle."""
    mod = f32_model(lgssm.dense_model(d, seed=5))
    _, y = lgssm.generate_data(mod, T, batch, seed=48)
    yd = dev(y)
    ctx.set_option("no_umma", 0)
    a = ctx.lgssm(yd, **_kw(mod), smooth=True, cov_shared_out=True)
    fa = ctx.lgssm(yd, **_kw(mod), smooth=False, transition_first=True, cov_shared_out=True)
    ctx.set_option("no_umma", 1)
    b = ctx.lgssm(yd, **_kw(mod), smooth=True, cov_shared_out=True)
    fb = ctx.lgssm(yd, **_kw(mod), smooth=False, transition_first=True, cov_shared_out=True)
    assert rel_l2(a["mean"].cpu().numpy(), b["mean"].cpu().numpy()) < 5e-6
    assert rel_l2(fa["mean"].cpu().numpy(), fb["mean"].cpu().numpy()) < 5e-6
    ref = lgssm.smooth_reference_schedule(y, **mod)
    assert rel_l2(a["mean"].cpu().numpy(), ref["mean"]) < TOL_MEAN
    assert rel_l2(fa["mean"].cpu().numpy(), lgssm.filter_streaming(y, **mod)["mean"]) < TOL_MEAN


@pytest.mark.parametrize("d,T,batch,tf", [(8, 60, 45, False), (16, 130, 70, True), (32, 90, 33, False), (64, 120, 130, True)])
def test_large_state_evidence(ctx, monkeypatch, d, T, batch, tf):
    """neg_log_evidence (= Bethe free energy on the tree) of the large-state family: filter-mode sweep + time-parallel
    whitened-innovation kernels; smoothing and filtering calls, both sweep implementations, prior on x[1] or one
    transition earlier."""
    mod = f32_model(lgssm.dense_model(d, seed=9))
    _, y = lgssm.generate_data(mod, T, batch, seed=49)
    ref = lgssm.smooth_reference_schedule(y, **mod, transition_first=tf)
    for no_umma in ("0", "1"):
        ctx.set_option("no_umma", int(no_umma))
        r = ctx.lgssm(dev(y), **_kw(mod), smooth=True, want_evidence=True, transition_first=tf, cov_shared_out=True)
        n = r["neg_log_evidence"].cpu().numpy().astype(np.float64)
        assert np.max(np.abs(n - ref["neg_log_evidence"]) / np.abs(ref["neg_log_evidence"])) < TOL_NLE
        assert rel_l2(r["mean"].cpu().numpy(), ref["mean"]) < TOL_MEAN
        f = ctx.lgssm(dev(y), **_kw(mod), smooth=False, want_evidence=True, transition_first=tf, cov_shared_out=True)
        nf = f["neg_log_evidence"].cpu().numpy().astype(np.float64)
        assert np.max(np.abs(nf - ref["neg_log_evidence"]) / np.abs(ref["neg_log_evidence"])) < TOL_NLE
        assert rel_l2(f["mean"].cpu().numpy(), ref["filt_mean"]) < TOL_MEAN


@pytest.mark.parametrize("d", [4, 16])
def test_non_spd_shared_model_is_reported(ctx, rx, d):
    """A shared model whose covariance recursion hits a non-positive Cholesky pivot must not come back as OK
    (ADVICE r1): synchronous calls return RXG_ERR_NOT_SPD, status[] carries it per chain, and a deferred
    (asynchronous) call reports it at rxg_sync.  The reference throws from cholinv here."""
    mod = f32_model(lgssm.notebook_model(4) if d == 4 else lgssm.dense_model(d))
    _, y = lgssm.generate_data(mod, 30, 40, seed=3)
    bad = dict(_kw(mod))
    bad["Q"] = -np.asarray(mod["Q"]) * 1e3          # innovation covariance B S B' + Q indefinite
    with pytest.raises(rx._lib.RxGaussError) as e:
        ctx.lgssm(dev(y), **bad, smooth=True)
    assert e.value.code == rx._lib.RXG_ERR_NOT_SPD
    with pytest.raises(rx._lib.RxGaussError) as e:
        ctx.lgssm(dev(y), **bad, smooth=True, asynchronous=True)
        ctx.sync()
    assert e.value.code == rx._lib.RXG_ERR_NOT_SPD
    st = torch.zeros(40, dtype=torch.int32, device="cuda")
    try:
        ctx.lgssm(dev(y), **bad, smooth=False, want_status=True, out_status=st)
    except rx._lib.RxGaussError:
        pass
    assert st.cpu().tolist() == [rx._lib.RXG_ERR_NOT_SPD] * 40
    # and a good model right after is clean again
    r = ctx.lgssm(dev(y), **_kw(mod), smooth=True, want_status=True)
    assert int(r["status"].abs().sum()) == 0


def test_context_validates_arrays(ctx):
    """Wrong dtype / layout / device must raise instead of handing a garbage pointer to the library (ADVICE r1)."""
    mod = f32_model(lgssm.notebook_model(4))
    _, y = lgssm.generate_data(mod, 20, 16, seed=4)
    yd = dev(y)
    with pytest.raises(ValueError):
        ctx.lgssm(yd.permute(0, 2, 1).contiguous().permute(0, 2, 1), **_kw(mod))          # non-contiguous view
    with pytest.raises(ValueError):
        ctx.lgssm(yd.double(), **_kw(mod))
    with pytest.raises(ValueError):
        ctx.lgssm(yd, **_kw(mod), mask=torch.ones(20, 16, dtype=torch.uint8))              # host mask, device y
    with pytest.raises(ValueError):
        ctx.lgssm(yd, **_kw(mod), out_mean=torch.empty(20, 4, 15, device="cuda"))
    with pytest.raises(ValueError):
        ctx.lgssm(yd, **_kw(mod), out_cov=torch.empty(20, 4, 4, device="cuda"))           # table shape without the flag


@pytest.mark.parametrize("d,m", [(4, 4), (2, 2), (3, 3), (4, 2), (1, 1), (2, 1), (4, 1)])
def test_time_segmented_sweep(ctx, d, m):
    """lgssm_seg_kernel (sweep_variant 3: parallel in time inside a chain tile; experimental, see the kernel header) against the oracle and the sequential-in-time sweep: segment boundaries (T = 1, 15, 16, 17, 33, 1000),
    ragged chain tiles, transition offset, prior one transition before the first datum, per-chain prior means."""
    rng = np.random.default_rng(300 + 10 * d + m)
    Aq, _ = np.linalg.qr(rng.standard_normal((d, d)))
    mod = f32_model(dict(A=0.95 * Aq, B=rng.standard_normal((m, d)), P=0.2 * np.eye(d), Q=1.5 * np.eye(m),
                         m0=rng.standard_normal(d), S0=5.0 * np.eye(d)))
    u = (0.3 * rng.standard_normal(d)).astype(np.float32)
    for T, batch in [(1, 33), (15, 64), (16, 70), (17, 31), (33, 203), (1000, 96)]:
        _, y = lgssm.generate_data(mod, T, batch, seed=41 + T)
        for kw in (dict(), dict(u=u), dict(transition_first=True), dict(u=u, transition_first=True)):
            ref = lgssm.smooth_reference_schedule(y, **mod, **{k: (v.astype(np.float64) if k == "u" else v) for k, v in kw.items()})
            ctx.set_option("sweep_variant", 0)
            base = ctx.lgssm(dev(y), **_kw(mod), smooth=True, **kw)
            for variant in (3,):
                ctx.set_option("sweep_variant", variant)
                r = ctx.lgssm(dev(y), **_kw(mod), smooth=True, **kw)
                check(r, ref, nle=False)
                assert rel_l2(r["mean"].cpu().numpy(), base["mean"].cpu().numpy()) < 2e-6
                assert torch.equal(r["cov"], base["cov"])            # the covariances come from the same table entries
        ctx.set_option("sweep_variant", 3)
        rs = ctx.lgssm(dev(y), **_kw(mod), smooth=True, cov_shared_out=True)
        assert rs["cov"].shape == (T, d, d)
        assert rel_l2(rs["mean"].cpu().numpy(), lgssm.smooth_reference_schedule(y, **mod)["mean"]) < TOL_MEAN


def test_time_segmented_sweep_full_size(ctx):
    """Headline size (d = m = 4, T = 1000, batch 65 536): the time-segmented kernel against the sequential sweep on
    every chain, and sampled chains against the oracle."""
    mod = f32_model(lgssm.notebook_model(4))
    T, batch = 1000, 65536
    g = torch.Generator(device="cuda").manual_seed(77)
    y = torch.randn(T, 4, batch, device="cuda", generator=g) * 3.3
    ctx.set_option("sweep_variant", 0)
    base = ctx.lgssm(y, **_kw(mod), smooth=True)
    for variant in (3,):
        ctx.set_option("sweep_variant", variant)
        r = ctx.lgssm(y, **_kw(mod), smooth=True)
        num = (r["mean"] - base["mean"]).double().norm().item()
        assert num / base["mean"].double().norm().item() < 2e-6
        assert torch.equal(r["cov"], base["cov"])
    idx = [0, 31, 32, 40000, 65535]
    ref = lgssm.smooth_reference_schedule(y[:, :, idx].cpu().numpy(), **mod)
    assert rel_l2(r["mean"][:, :, idx].cpu().numpy(), ref["mean"]) < TOL_MEAN


def test_large_state_d64_full_length(ctx):
    """BASELINE configs[2] at its real length (d = 64, T = 1000): the 3xTF32 tensor-core recursion against the fp64
    oracle over all 1000 steps (round 1 stopped at T = 300), per-chain covariance output included."""
    mod = f32_model(lgssm.dense_model(64))
    T, batch = 1000, 6
    _, y = lgssm.generate_data(mod, T, batch, seed=64)
    ref = lgssm.smooth_reference_schedule(y, **mod)
    r = ctx.lgssm(dev(y), **_kw(mod), smooth=True, want_evidence=True)
    em = rel_l2(r["mean"].cpu().numpy(), ref["mean"])
    ec = rel_l2(r["cov"].cpu().numpy(), ref["cov"])
    print("d=64 T=1000: mean relL2", em, "cov relF", ec)
    assert em < TOL_MEAN and ec < TOL_COV
    check(r, ref)
    assert torch.equal(r["cov"][..., 0], r["cov"][..., batch - 1])


@pytest.mark.parametrize("d,m", [(4, 4), (2, 1), (5, 3), (16, 16)])
def test_shared_missing_data_pattern_stays_on_gain_table_path(ctx, d, m):
    """RXG_MASK_SHARED: one missing-data pattern for all chains (host array [T]).  The covariances stay chain independent,
    so the gain tables handle it (missing step = pure transition) and the mean sweep is unchanged; result = the per-chain
    mask path with the pattern broadcast = the oracle.  Time-parallel scan and sequential gain kernels, smoothing and
    filtering with evidence, first / last step missing, T > 1024 (several steps per scan thread)."""
    rng = np.random.default_rng(77 + d)
    mod = _random_model(rng, d, m) if (d, m) != (4, 4) else f32_model(lgssm.notebook_model(4))
    for T, batch in ((40, 70), (1300, 6)) if d <= 5 else ((24, 9),):
        _, y = lgssm.generate_data(mod, T, batch, seed=5 + T)
        tm = (rng.random(T) > 0.3).astype(np.uint8)
        tm[0] = 0; tm[-1] = 0; tm[1] = 1
        full = np.repeat(tm[:, None], batch, axis=1)
        ref = lgssm.smooth_reference_schedule(y, **mod, mask=full)
        for seq in (0, 1):
            ctx.set_option("gain_seq", seq)
            r = ctx.lgssm(dev(y), **_kw(mod), smooth=True, mask=tm, want_evidence=True)
            check(r, ref)
            f = ctx.lgssm(dev(y), **_kw(mod), smooth=False, mask=tm, want_evidence=True)
            check(f, ref, smooth=False)
        ctx.set_option("gain_seq", 0)
        if d <= 5:
            assert torch.equal(r["cov"][..., 0], r["cov"][..., batch - 1])        # still chain independent
            rp = ctx.lgssm(dev(y), **_kw(mod), smooth=True, mask=dev(full, torch.uint8))
            assert rel_l2(r["mean"].cpu().numpy(), rp["mean"].cpu().numpy()) < 2 * TOL_MEAN
