"""Known per-step inputs on the GPU: every family of the batched LGSSM sweeps, every chain gated at the unchanged
TOL_MEAN / TOL_COV / TOL_NLE against the fp64 references of test_inputs.py.

Routes (csrc/rxg_lgssm*.cu): a shared sequence (RXG_U_SEQ_SHARED) goes into the gain tables' offset terms (register
families) or the host trajectory of the linearity route (large-state family); a per-chain sequence (RXG_U_SEQ_CHAIN) is
streamed by its own `lgssm_shared_kernel` instantiation (register families) or removed by linearity with a per-chain
trajectory (large-state family); the per-chain kernels read u[t] inside the step.
"""
import ctypes
import itertools

import numpy as np
import pytest
import torch

from oracle import lgssm
from test_inputs import forecast_reference, input_reference, input_sequence, kalman_rts_inputs, per_chain_models
from test_shared_sweep_variants import (MATRIX_T, _eq, _kw, ck_eligible, covariance_side, gate_cov, gate_mean, gate_nle,
                                        pattern, random_model, simulate)
from util import f32_model

REGISTER = [(1, 1), (2, 1), (2, 2), (3, 3), (4, 1), (4, 2), (4, 4), (6, 6), (3, 2), (5, 3)]
LARGE = [(8, 8), (16, 16), (64, 64), (12, 7), (33, 20)]


def _run(ctx, y, mod, useq, *, cpt=0, variant=0, smooth=True, evid=False, tf=False, tm=None, cov_shared=False, u=None,
         **kw):
    ctx.set_option("force_cpt", cpt)
    ctx.set_option("sweep_variant", variant)
    inputs = None
    if useq is not None:
        inputs = torch.as_tensor(useq, device="cuda") if useq.ndim == 3 else useq
    return ctx.lgssm(y, **_kw(mod), u=u, inputs=inputs, smooth=smooth, mask=tm, want_evidence=evid, transition_first=tf,
                     cov_shared_out=cov_shared, **kw)


def _gate(cat, case, r, ref, nb, evid):
    gate_mean(cat, case, r["mean"], ref["mean"][..., :nb])
    if evid:
        gate_nle(cat, case, r["neg_log_evidence"], ref["nle"][:nb])


# ====================================================================================== register families, shared model
@pytest.mark.gpu
@pytest.mark.parametrize("T", MATRIX_T)
@pytest.mark.parametrize("d,m", REGISTER)
def test_register_matrix(ctx, d, m, T):
    """Shared / per-chain sequence x smoothing / filtering x evidence x transition_first x no / shared mask, at CPT 1,
    CPT 2 (checkpoint at d <= 4) and CPT 2 stash, batch 70 and 71 (odd: the CPT 1 fallback)."""
    mod = random_model(d, m, seed=1000 + 16 * d + m)         # the data of test_variant_matrix
    y_np = simulate(mod, T, 71, seed=31 * T + d + m)
    tm = pattern(T)
    ck = ck_eligible(d, m)
    useqs = dict(shared=input_sequence(T, d, seed=T + d), chain=input_sequence(T, d, seed=T + m, nb=71))
    for kind, smooth, evid, tf, use_mask in itertools.product(("shared", "chain"), (True, False), (False, True),
                                                              (False, True), (False, True)):
        case = (f"d={d} m={m} T={T} {kind} {'smooth' if smooth else 'filter'} evid={int(evid)} tf={int(tf)} "
                f"mask={int(use_mask)}")
        tmk = tm if use_mask else None
        y71 = torch.as_tensor(y_np, device="cuda")
        us = useqs[kind]
        ref = input_reference(mod, y71.cpu(), us, smooth=smooth, transition_first=tf, tmask=tmk)
        y70 = y71[..., :70].contiguous()
        us70 = us if kind == "shared" else np.ascontiguousarray(us[..., :70])
        kw = dict(smooth=smooth, evid=evid, tf=tf, tm=tmk)
        r1 = _run(ctx, y70, mod, us70, cpt=1, **kw)
        _gate("register", case + " cpt=1", r1, ref, 70, evid)
        gate_cov("register", case, r1["cov"], ref["cov"])
        r2 = _run(ctx, y70, mod, us70, cpt=2, **kw)
        _gate("register", case + " cpt=2", r2, ref, 70, evid)
        outs = [r1, r2]
        if smooth and ck:
            rs = _run(ctx, y70, mod, us70, cpt=2, variant=1, **kw)
            _gate("register", case + " cpt=2 stash", rs, ref, 70, evid)
            outs.append(rs)
        # covariances do not see the inputs
        r0 = _run(ctx, y70, mod, None, cpt=2, **kw)
        for r in outs:
            _eq(r["cov"], r0["cov"], "covariances with / without inputs", case)
        if not evid:
            for r in outs[1:]:
                _eq(r1["mean"], r["mean"], "mean across CPT / stash / CK", case)
        else:
            for r in outs[1:]:
                _eq(r1["neg_log_evidence"], r["neg_log_evidence"], "nle across CPT / stash / CK", case)
        if smooth and not evid:      # the time-segmented sweep is not extended: the lock-step kernel runs
            r3 = _run(ctx, y70, mod, us70, cpt=2, variant=3, **kw)
            _eq(r3["mean"], r2["mean"], "sweep_variant 3 vs 0 with inputs", case)
        ro = _run(ctx, y71, mod, us, cpt=2, **kw)
        _gate("register", case + " batch=71", ro, ref, 71, evid)
        _eq(ro["mean"][..., :70], r1["mean"], "odd batch (CPT 1 fallback) vs CPT 1", case)


def _constant_vs_offset(ctx, d, m, T, cpt=0):
    mod = random_model(d, m, seed=6000 + 16 * d + m)
    y = torch.as_tensor(simulate(mod, T, 70, seed=d + m), device="cuda")
    u = (0.5 * np.random.default_rng(d + m).standard_normal(d)).astype(np.float32)
    useq = np.tile(u, (T, 1))
    for smooth, evid, tf in itertools.product((True, False), (False, True), (False, True)):
        case = f"d={d} m={m} T={T} smooth={int(smooth)} evid={int(evid)} tf={int(tf)}"
        a = _run(ctx, y, mod, useq, cpt=cpt, smooth=smooth, evid=evid, tf=tf)
        b = _run(ctx, y, mod, None, cpt=cpt, smooth=smooth, evid=evid, tf=tf, u=u)
        _eq(a["mean"], b["mean"], "constant-row sequence vs constant u (mean)", case)
        _eq(a["cov"], b["cov"], "constant-row sequence vs constant u (cov)", case)
        _eq(a["neg_log_evidence"], b["neg_log_evidence"], "constant-row sequence vs constant u (nle)", case)


@pytest.mark.gpu
@pytest.mark.parametrize("d,m", REGISTER + LARGE)
def test_constant_sequence_equals_constant_offset(ctx, d, m):
    """A shared sequence with constant rows is bit for bit the constant-u call (gain tables / host trajectory)."""
    for cpt in ((1, 2) if (d, m) in REGISTER else (0,)):
        _constant_vs_offset(ctx, d, m, 25, cpt)


@pytest.mark.gpu
@pytest.mark.parametrize("d,m", [(1, 1), (4, 4), (6, 6), (5, 3), (16, 16), (12, 7)])
def test_chain_sequence_repeating_the_shared_one(ctx, d, m):
    """A per-chain sequence that repeats the shared sequence in every chain agrees with the shared call."""
    mod = random_model(d, m, seed=6500 + d)
    T = 29
    y = torch.as_tensor(simulate(mod, T, 70, seed=d), device="cuda")
    us = input_sequence(T, d, seed=d)
    uc = np.ascontiguousarray(np.repeat(us[..., None], 70, axis=2))
    ref = input_reference(mod, y.cpu(), us, transition_first=True)
    for evid in (False, True):
        a = _run(ctx, y, mod, us, evid=evid, tf=True)
        b = _run(ctx, y, mod, uc, evid=evid, tf=True)
        for r in (a, b):
            _gate("repeat", f"d={d} m={m} evid={int(evid)}", r, ref, 70, evid)
        _eq(a["cov"], b["cov"], "covariances shared vs per-chain sequence", f"d={d}")


# ====================================================================================== large-state family
@pytest.mark.gpu
@pytest.mark.parametrize("T", [1, 5, 13, 25])
@pytest.mark.parametrize("d,m", LARGE)
def test_large_family(ctx, d, m, T):
    """The linearity route: shared (host trajectory) and per-chain (input_traj_kernel) sequences, smoothing / filtering
    x evidence x transition_first; covariances equal to the call without inputs."""
    mod = random_model(d, m, seed=7000 + d + m)
    y = torch.as_tensor(simulate(mod, T, 70, seed=T + d), device="cuda")
    useqs = dict(shared=input_sequence(T, d, seed=T), chain=input_sequence(T, d, seed=T + 1, nb=70))
    for kind, smooth, evid, tf in itertools.product(("shared", "chain"), (True, False), (False, True), (False, True)):
        case = f"d={d} m={m} T={T} {kind} {'smooth' if smooth else 'filter'} evid={int(evid)} tf={int(tf)}"
        ref = input_reference(mod, y.cpu(), useqs[kind], smooth=smooth, transition_first=tf)
        r = _run(ctx, y, mod, useqs[kind], smooth=smooth, evid=evid, tf=tf)
        _gate("large", case, r, ref, 70, evid)
        gate_cov("large", case, r["cov"], ref["cov"])
        r0 = _run(ctx, y, mod, None, smooth=smooth, evid=evid, tf=tf)
        _eq(r["cov"], r0["cov"], "covariances with / without inputs", case)


# ====================================================================================== per-chain paths
@pytest.mark.gpu
@pytest.mark.parametrize("d,m", REGISTER + [(8, 8), (12, 7), (33, 20)])
@pytest.mark.parametrize("path", ["per_chain_model", "per_chain_mask", "forced"])
def test_per_chain_paths(ctx, d, m, path):
    """lgssm_chain_kernel (d <= 6) and lgssm_generic_chain_kernel (other shapes) with u[t] read inside the step: a
    per-chain model, a per-chain mask, or the forced per-chain path; shared and per-chain sequences."""
    nb = 70
    mod = random_model(d, m, seed=8000 + 16 * d + m)
    rng = np.random.default_rng(d * m)
    for T in (1, 13, 25):
        y = torch.as_tensor(simulate(mod, T, nb, seed=T + d), device="cuda")
        mods = per_chain_models(mod, nb)
        kw = {}
        mask = None
        if path == "per_chain_model":
            # chain-dependent A: the shared model with a per-chain scale on A
            sc = torch.as_tensor(0.8 + 0.2 * rng.random(nb))
            mods["A"] = mods["A"] * sc[:, None, None]
            pc = {k: v.permute(*range(1, v.dim()), 0).contiguous().float().cuda() for k, v in mods.items()}
            kw = dict(per_chain_model=True, A=pc["A"], B=pc["B"], P=pc["P"], Q=pc["Q"], m0=pc["m0"], S0=pc["S0"])
        elif path == "per_chain_mask":
            mask = (rng.random((T, nb)) > 0.3).astype(np.uint8)
            kw = dict(mask=torch.as_tensor(mask, device="cuda"))
        else:
            kw = dict(force_per_chain_path=True)
        for kind, smooth, tf in itertools.product(("shared", "chain"), (True, False), (False, True)):
            case = f"{path} d={d} m={m} T={T} {kind} {'smooth' if smooth else 'filter'} tf={int(tf)}"
            us = input_sequence(T, d, seed=T + 3) if kind == "shared" else input_sequence(T, d, seed=T + 4, nb=nb)
            ref = kalman_rts_inputs(mods, y.cpu(), us, mask=mask, smooth=smooth, transition_first=tf)
            inputs = torch.as_tensor(us, device="cuda") if kind == "chain" else us
            args = dict(_kw(mod), **{k: v for k, v in kw.items() if k in ("A", "B", "P", "Q", "m0", "S0")})
            rest = {k: v for k, v in kw.items() if k not in ("A", "B", "P", "Q", "m0", "S0")}
            r = ctx.lgssm(y, **args, inputs=inputs, smooth=smooth, want_evidence=True, transition_first=tf, **rest)
            r0 = ctx.lgssm(y, **args, smooth=smooth, want_evidence=False, transition_first=tf, **rest)
            gate_mean("per-chain", case, r["mean"], ref["mean"])
            gate_nle("per-chain", case, r["neg_log_evidence"], ref["nle"])
            g = torch.linalg.norm((r["cov"].double().cpu() - ref["cov"]).flatten(0, 2), dim=0) / \
                torch.linalg.norm(ref["cov"].flatten(0, 2), dim=0)
            from util import TOL_COV
            assert float(g.max()) < TOL_COV, f"{case}: covariance of chain {int(g.argmax())} off by {float(g.max()):.2e}"
            _eq(r["cov"], r0["cov"], "covariances with / without inputs", case)


# ====================================================================================== streaming, predictions, infer
@pytest.mark.gpu
@pytest.mark.parametrize("d,m", [(1, 1), (4, 4), (6, 6), (5, 3), (16, 16)])
@pytest.mark.parametrize("kind", ["shared", "chain"])
def test_streaming_chunks_with_inputs(ctx, rx, d, m, kind):
    """Chunks of the streaming engine with their inputs ({"y": ..., "u": ...}) match one filtering call."""
    mod = random_model(d, m, seed=9000 + d)
    T, nb = 37, 70
    y = torch.as_tensor(simulate(mod, T, nb, seed=d), device="cuda")
    us = input_sequence(T, d, seed=d + 1, nb=None if kind == "shared" else nb)
    whole = ctx.lgssm(y, **_kw(mod), inputs=torch.as_tensor(us, device="cuda") if kind == "chain" else us, smooth=False,
                      transition_first=True, want_evidence=True)
    ref = input_reference(mod, y.cpu(), us, smooth=False, transition_first=True)
    gate_mean("streaming", f"d={d} {kind} whole", whole["mean"], ref["mean"])
    from rxinfer_jl_b200 import inference as I
    model = I.linear_gaussian_ssm_filtering(A=mod["A"], B=mod["B"], P=mod["P"], Q=mod["Q"], x0=(mod["m0"], mod["S0"]))
    eng = I.infer(model=model, datastream=None, autoupdates=True, batch=nb, keephistory=T, historyvars=["x_t"],
                  free_energy=True, context=ctx)
    for a, b in ((0, 12), (12, 13), (13, 37)):
        uc = us[a:b] if kind == "shared" else torch.as_tensor(np.ascontiguousarray(us[a:b]), device="cuda")
        eng.push({"y": y[a:b].contiguous(), "u": uc})
    got = torch.cat([p.mu for p in eng._hist["x_t"]])
    gate_mean("streaming", f"d={d} {kind} chunks", got, ref["mean"])
    gate_mean("streaming", f"d={d} {kind} chunks vs whole", got, whole["mean"].double())


@pytest.mark.gpu
@pytest.mark.parametrize("d,m", [(2, 1), (4, 4), (3, 2), (16, 16), (12, 7)])
@pytest.mark.parametrize("kind", ["shared", "chain"])
@pytest.mark.parametrize("per_chain_model", [False, True])
def test_predict_forecasts_with_inputs(ctx, d, m, kind, per_chain_model):
    """Forecast k = 1..H steps with row T + k - 1 of the inputs (== the smoother on y padded with H missing steps); the
    posteriors are those of the smoothing call with the first T rows."""
    mod = random_model(d, m, seed=9500 + d + m)
    T, H, nb = 21, 5, 70
    y = torch.as_tensor(simulate(mod, T, nb, seed=d + m), device="cuda")
    us = input_sequence(T + H, d, seed=3, nb=None if kind == "shared" else nb)
    inputs = us if kind == "shared" else torch.as_tensor(us, device="cuda")
    kw = dict(_kw(mod))
    if per_chain_model:
        pc = {k: v.permute(*range(1, v.dim()), 0).contiguous().float().cuda() for k, v in per_chain_models(mod, nb).items()}
        kw = dict(A=pc["A"], B=pc["B"], P=pc["P"], Q=pc["Q"], m0=pc["m0"], S0=pc["S0"])
    r = ctx.lgssm_predict(y, **kw, horizon=H, inputs=inputs, per_chain_model=per_chain_model)
    case = f"d={d} m={m} {kind} per_chain_model={int(per_chain_model)}"
    yp = torch.cat([y.cpu(), torch.zeros(H, m, nb)])
    mask = np.ones((T + H, nb), np.uint8); mask[T:] = 0
    pad = kalman_rts_inputs(per_chain_models(mod, nb), yp, us, mask=mask)
    gate_mean("predict", case + " posterior", r["mean"], pad["mean"][:T])
    gate_mean("predict", case + " forecast means", r["fc_mean"], pad["mean"][T:])
    fm, _ = forecast_reference(mod, r["mean"][-1].cpu().numpy(), r["cov"][-1].cpu().numpy(),
                               us[T:] if kind == "shared" else us[T:], H)
    gate_mean("predict", case + " forecast means vs forecast recursion", r["fc_mean"], torch.as_tensor(fm))
    B = torch.as_tensor(mod["B"], dtype=torch.float64)
    gate_mean("predict", case + " forecast observations", r["pred_mean"][T:], torch.einsum("kd,hdb->hkb", B, pad["mean"][T:]))
    base = ctx.lgssm(y, **kw, inputs=inputs[:T] if kind == "shared" else inputs[:T].contiguous(),
                     per_chain_model=per_chain_model)
    _eq(r["mean"], base["mean"], "predict posteriors vs smoothing call", case)


@pytest.mark.gpu
def test_infer_with_inputs(ctx, rx):
    """infer(data = {"y": y, "u": inputs}) for the smoothing and filtering models, and with predictions."""
    from rxinfer_jl_b200 import inference as I
    mod = random_model(4, 4, seed=11)
    T, H, nb = 30, 3, 70
    y = torch.as_tensor(simulate(mod, T, nb, seed=2), device="cuda")
    us = input_sequence(T + H, 4, seed=5, nb=nb)
    uc = torch.as_tensor(us, device="cuda")
    sm = I.linear_gaussian_ssm_smoothing(A=mod["A"], B=mod["B"], P=mod["P"], Q=mod["Q"], x0=(mod["m0"], mod["S0"]))
    r = I.infer(model=sm, data={"y": y, "u": uc[:T].contiguous()}, context=ctx)
    gate_mean("infer", "smoothing", r.posteriors["x"].mu, input_reference(mod, y.cpu(), us[:T])["mean"])
    fl = I.linear_gaussian_ssm_filtering(A=mod["A"], B=mod["B"], P=mod["P"], Q=mod["Q"], x0=(mod["m0"], mod["S0"]))
    r = I.infer(model=fl, data={"y": y, "u": us[:T, :, 0].copy()}, context=ctx)
    gate_mean("infer", "filtering", r.history["x_t"].mu,
              input_reference(mod, y.cpu(), us[:T, :, 0], smooth=False, transition_first=True)["mean"])
    smh = I.linear_gaussian_ssm_smoothing(A=mod["A"], B=mod["B"], P=mod["P"], Q=mod["Q"], x0=(mod["m0"], mod["S0"]), horizon=H)
    r = I.infer(model=smh, data={"y": y, "u": uc}, predictvars=I.KeepLast(), context=ctx)
    assert set(r.predictions) == {"y"}
    assert r.posteriors["x"].mu.shape == (T + H, 4, nb)


# ====================================================================================== full size
@pytest.mark.gpu
def test_full_size_chain_sequence_every_chain(ctx):
    """The config-2 call (notebook model, d = m = 4, T = 1000, 65 536 chains) with a per-chain input sequence,
    checkpointing (the default dispatch) and evidence: every chain against the fp64 reference."""
    T, nb = 1000, 65536
    mod = f32_model(lgssm.notebook_model(4))
    g = torch.Generator(device="cuda").manual_seed(4242)
    y = torch.randn(T, 4, nb, device="cuda", generator=g) * 3.3
    u = torch.randn(T, 4, nb, device="cuda", generator=g) * 0.5
    r = ctx.lgssm(y, **_kw(mod), inputs=u, want_evidence=True)
    cs = covariance_side(mod, T)
    ref = input_reference(mod, y, u, cs=cs)
    gate_mean("full", "chain sequence ck evid", r["mean"], ref["mean"])
    gate_nle("full", "chain sequence ck evid", r["neg_log_evidence"], ref["nle"])
    gate_cov("full", "chain sequence ck evid", r["cov"], ref["cov"])
    del r, ref, y, u
    torch.cuda.empty_cache()


# ====================================================================================== refusals
def _raw_smooth(ctx, y, mod, u_ptr, flags):
    from rxinfer_jl_b200 import _lib as L
    T, m, nb = y.shape
    d = mod["A"].shape[0]
    keep = [np.ascontiguousarray(mod[k], np.float32) for k in ("A", "B", "P", "Q", "m0", "S0")]
    mean = torch.empty(T, d, nb, device="cuda"); cov = torch.empty(T, d, d, nb, device="cuda")
    fp = lambda t: L.as_fp(t.data_ptr())
    return ctx.lib.rxg_lgssm_smooth_f32(ctx.h, d, m, T, nb, *[k.ctypes.data_as(L.fp) for k in keep], u_ptr, fp(y),
                                        ctypes.cast(ctypes.c_void_p(None), L.u8p), fp(mean), fp(cov), L.as_fp(0),
                                        ctypes.cast(ctypes.c_void_p(None), L.i32p), flags)


@pytest.mark.gpu
def test_refusals(ctx, rx):
    from rxinfer_jl_b200 import _lib as L
    mod = random_model(4, 4, seed=1)
    T, nb = 9, 8
    y = torch.as_tensor(simulate(mod, T, nb, seed=1), device="cuda")
    us = np.ascontiguousarray(input_sequence(T, 4, seed=1))
    up = us.ctypes.data_as(L.fp)
    assert _raw_smooth(ctx, y, mod, up, L.PTR_DEVICE | L.U_SEQ_SHARED | L.U_SEQ_CHAIN) == L.RXG_ERR_BAD_ARG
    assert _raw_smooth(ctx, y, mod, L.as_fp(0), L.PTR_DEVICE | L.U_SEQ_SHARED) == L.RXG_ERR_BAD_ARG      # no sequence
    assert _raw_smooth(ctx, y, mod, up, L.PTR_DEVICE | L.U_SEQ_SHARED) == 0
    # a per-chain sequence with host pointers
    uc = torch.as_tensor(input_sequence(T, 4, seed=2, nb=nb), device="cuda")
    with pytest.raises(L.RxGaussError) as e:
        ctx.lgssm(y.cpu(), **_kw(mod), inputs=uc)
    assert e.value.code == L.RXG_ERR_UNSUPPORTED
    # the fused gather refuses both flags before anything runs (no peer group is needed to get there)
    keep = [np.ascontiguousarray(mod[k], np.float32) for k in ("A", "B", "P", "Q", "m0", "S0")]
    for f in (L.U_SEQ_SHARED, L.U_SEQ_CHAIN):
        rc = ctx.lib.rxg_lgssm_smooth_gather_f32(ctx.h, 4, 4, T, nb, *[k.ctypes.data_as(L.fp) for k in keep], up,
                                                 L.as_fp(y.data_ptr()), ctypes.cast(ctypes.c_void_p(None), L.u8p), None, None,
                                                 L.as_fp(0), ctypes.cast(ctypes.c_void_p(None), L.i32p), L.PTR_DEVICE | f)
        assert rc == L.RXG_ERR_UNSUPPORTED
