#!/usr/bin/env python
"""Secondary measurements (not the driver's bench contract): the other BASELINE.json configs and
the per-rule kernels, one JSON line each.  Device-resident data, CUDA events, >= 3 warm-ups.

  python bench_extra.py [--which per_chain,filter,hgf,rules,vmp,scaling_T]
  python bench_extra.py --which predict      (opt-in: observation predictions / forecasts after the smoother)
  python bench_extra.py --which inputs       (opt-in: known per-step inputs u[t], shared and per-chain sequences)
  python bench_extra.py --which vmp_wishart  (opt-in: Wishart-precision VMP around the smoother vs the composed path)
  python bench_extra.py --which vmp_noise    (opt-in: learned process precision, alone and with the observation precision)
  python bench_extra.py --which vmp_transition (opt-in: learned transition matrix, alone and with the noise precisions)
  python bench_extra.py --which gmm          (opt-in: Gaussian-mixture VMP, d = 2 / K = 3 and d = 4 / K = 8)
  python bench_extra.py --which hmm          (opt-in: hidden Markov model VMP, K = M = 3 and K = 8 / M = 16)
  python bench_extra.py --which hmm_gauss    (opt-in: Gaussian-emission HMM VMP, K = 3 / d = 2 and K = 8 / d = 4)
  python bench_extra.py --which binomial     (opt-in: binomial regression VMP, both kernels, and the grid that places the
                                             automatic choice between them)
  python bench_extra.py --which multinomial  (opt-in: multinomial regression VMP, whole data sets and online, per-kernel
                                             times, data-pass bandwidth and fp64 FMA rate)
  python bench_extra.py --which hgf_learn    (opt-in: HGF with learned kappa, omega, T = 1000, 20 iterations)
  python bench_extra.py --which delta        (opt-in: Delta node: the paper's pendulum stream, the d = 4 tracker smoother)
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
import rxinfer_jl_b200 as rx  # noqa: E402
from bench import dense_model_f32, notebook_model_d2_f32, notebook_model_f32, peaks  # noqa: E402


def timed(fn, warm=3, reps=5):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def gpu_name_and_power_limit():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, plim = (x.strip() for x in out.split(",")[:2])
        return name, plim
    except Exception:
        return torch.cuda.get_device_name(0), "unknown"


def bench_predict(ctx, peak):
    """Smoother alone vs smoother + predictions (rxg_lgssm_smooth_predict_f32); the post-pass time is the difference of the
    two (CUDA events, same inputs, alternated).  Algorithmic bytes of the post-pass means: read y (4 m, observed steps only)
    and mu (4 d), write y_hat (4 m) per (chain, step); forecast rows read and write the state (8 d) and write y_hat (4 m)."""
    gname, plim = gpu_name_and_power_limit()
    g = torch.Generator(device="cuda").manual_seed(11)
    nb = notebook_model_f32()
    dn = dense_model_f32(64)
    cases = [("config-2 size, shared model, H = 0", nb, 1000, 65536, 0, None),
             ("config-2 size, shared model, H = 100, last 100 steps missing (shared mask)", nb, 1000, 65536, 100, "tail"),
             ("d = 64 dense model, H = 0 (left-GEMM route)", dn, 1000, 4096, 0, None)]
    for name, mod, T, batch, H, mk in cases:
        d, m = mod["A"].shape[0], mod["B"].shape[0]
        y = torch.randn(T, m, batch, device="cuda", generator=g) * 3.3
        mask = None
        if mk == "tail":
            mask = np.ones(T, dtype=np.uint8); mask[-100:] = 0
        args = [mod[k] for k in ("A", "B", "P", "Q", "m0", "S0")]
        smooth = lambda: ctx.lgssm(y, *args, mask=mask, cov_shared_out=mask is None)
        # with a mask the smoother writes per-chain covariances: there the post-pass is timed for the prediction means
        # only (no per-chain prediction or state-forecast covariance broadcast, state forecasts in library scratch)
        pred = lambda: ctx.lgssm_predict(y, *args, horizon=H, mask=mask, cov_shared_out=mask is None,
                                         want_pred_cov=mask is None, want_forecast_states=H > 0 and mask is None)
        ts, tp = [], []
        for _ in range(3):
            ts.append(timed(smooth)); tp.append(timed(pred))
        ms_s, ms_p = float(np.median(ts)), float(np.median(tp))
        nobs = T - (100 if mk == "tail" else 0)
        byts = 4 * batch * (nobs * (d + 2 * m) + (T - nobs) * (d + m) + H * (2 * d + m + d))
        post = ms_p - ms_s
        print(json.dumps({"what": "lgssm smooth + predictions: " + name, "d": d, "m": m, "T": T, "H": H, "batch": batch,
                          "smoother_ms": ms_s, "smoother_plus_predict_ms": ms_p, "postpass_ms": post,
                          "postpass_algorithmic_GB": byts / 1e9,
                          "postpass_frac_of_peak_hbm": (byts / (post * 1e-3)) / (peak * 1e9) if post > 0 else None,
                          "peak_hbm_gbs": peak, "gpu": gname, "power_limit": plim}), flush=True)
        del y
        torch.cuda.empty_cache()


def bench_inputs(ctx, peak):
    """Smoothing with known per-step inputs at config-2 size (notebook model, d = m = 4, T = 1000, 65 536 chains): no input,
    constant u, a shared sequence and a per-chain sequence (checkpoint and stash at CPT 2), each as kernel time (the
    sweep kernel's CUDA events, rxg_profile_last_ms) and call time; plus the d = 64 linearity route at batch 4096.
    Algorithmic bytes per (chain, step): read y (4 m) [+ u (4 d) for a per-chain sequence], write the smoothed mean (4 d)
    and covariance (4 d^2)."""
    gname, plim = gpu_name_and_power_limit()
    g = torch.Generator(device="cuda").manual_seed(12)
    nb = notebook_model_f32()
    dn = dense_model_f32(64)
    cases = [("config-2, no input", nb, 65536, None, 0), ("config-2, constant u", nb, 65536, "const", 0),
             ("config-2, shared sequence", nb, 65536, "shared", 0),
             ("config-2, per-chain sequence, CPT 2 checkpoint", nb, 65536, "chain", 0),
             ("config-2, per-chain sequence, CPT 2 stash", nb, 65536, "chain", 1),
             ("d = 64 dense, per-chain sequence (linearity route)", dn, 4096, "chain", 0),
             ("d = 64 dense, no input", dn, 4096, None, 0)]
    T = 1000
    for name, mod, batch, kind, variant in cases:
        d, m = mod["A"].shape[0], mod["B"].shape[0]
        y = torch.randn(T, m, batch, device="cuda", generator=g) * 3.3
        args = [mod[k] for k in ("A", "B", "P", "Q", "m0", "S0")]
        u = (0.3 * np.ones(d)).astype(np.float32) if kind == "const" else None
        inputs = None
        if kind == "shared":
            inputs = (0.3 * np.random.default_rng(1).standard_normal((T, d))).astype(np.float32)
        elif kind == "chain":
            inputs = torch.randn(T, d, batch, device="cuda", generator=g) * 0.3
        ctx.set_option("sweep_variant", variant)
        out_mean = torch.empty(T, d, batch, device="cuda")
        out_cov = torch.empty(T, d, d, batch, device="cuda")
        call = lambda: ctx.lgssm(y, *args, u=u, inputs=inputs, out_mean=out_mean, out_cov=out_cov)
        ctx.set_profiling(True)
        call_ms, kern_ms = [], []
        for _ in range(3):
            call_ms.append(timed(call))
            kms = []
            for _ in range(5):
                call()
                kms.append(ctx.profile_last_ms()[0])
            kern_ms.append(float(np.median(kms)))
        ctx.set_profiling(False)
        ctx.set_option("sweep_variant", 0)
        kms, cms = float(np.median(kern_ms)), float(np.median(call_ms))
        byts = 4 * T * batch * (m + d + d * d + (d if kind == "chain" else 0))
        print(json.dumps({"what": "lgssm smoothing with inputs: " + name, "d": d, "m": m, "T": T, "batch": batch,
                          "kernel_ms": kms, "call_ms": cms, "algorithmic_GB": byts / 1e9,
                          "algorithmic_bytes_per_chain_step": byts / (T * batch),
                          "kernel_frac_of_peak_hbm": (byts / (kms * 1e-3)) / (peak * 1e9),
                          "peak_hbm_gbs": peak, "gpu": gname, "power_limit": plim}), flush=True)
        del y, inputs, out_mean, out_cov
        torch.cuda.empty_cache()


def vmp_wishart_counts(d, m, masked, learn="Q"):
    """Algorithmic bytes and FLOPs per (chain, step, iteration) of one non-final iteration of the fused Wishart VMP kernel
    (lgssm_vmp_wishart_kernel), and the bytes of the same iteration on the composed path (per-chain smoother + a reduction
    over T).  Bytes: y is read in both directions (forward only when Q is known: the backward pass reads y for R_q); the
    filtered mean and the lower triangle of the filtered covariance are written (stash) and read back; a per-chain mask
    adds one byte per direction.  FLOPs: 2 x the FMAs of the step helpers (predict, update, RTS step), of the R_q
    accumulation (learned Q) and of the pair term of R_p (learned P: (I - A G) Ss (I - A G)' + A C A' + e e'), dense counts
    of rxg_linalg.cuh."""
    tri = lambda n: n * (n + 1) // 2
    stash = 4 * (d + tri(d))
    lq, lp = "Q" in learn, "P" in learn
    fused = (2 if lq else 1) * 4 * m + 2 * stash + ((2 if lq else 1) if masked else 0)
    composed = (4 * m + 2 * stash + 4 * (d + d * d) + (1 if masked else 0)) + (4 * m + 4 * d + 4 * d * d + (1 if masked else 0))
    predict = d * d + d ** 3 + tri(d) * d
    update = m * d * d + tri(m) * d + m ** 3 // 6 + d * m * m // 2 + m * d + m * m // 2 + d * m + tri(d) * m
    rts = d ** 3 + tri(d) * d + d ** 3 // 6 + d ** 3 // 2 + d ** 3 // 2 + tri(d) * d + d ** 3 + tri(d) * d + 2 * d * d
    acc = (m * d + m * m + m * d * d + tri(m) * d) if lq else 0
    pair = (3 * d ** 3 + 2 * tri(d) * d + d * d + tri(d)) if lp else 0
    return fused, composed, 2 * (predict + update + rts + acc + pair)


def _composed_wishart(ctx, y, mod, its, nu0, Psi0, W0, mask):
    """The path users compose without the fused entry: per-chain Context.lgssm with Q_b = inv(E[w_b]), a torch
    reduction over T and the Wishart update in torch (fp64)."""
    T, m, nb = y.shape
    dev = lambda M: torch.as_tensor(np.ascontiguousarray(np.broadcast_to(np.asarray(M, np.float32)[..., None],
                                                                          np.shape(M) + (nb,))), device="cuda")
    A, B, P, m0, S0 = (dev(mod[k]) for k in ("A", "B", "P", "m0", "S0"))
    Bd = torch.as_tensor(mod["B"], dtype=torch.float64, device="cuda")
    W = torch.as_tensor(W0, dtype=torch.float64, device="cuda").unsqueeze(0).repeat(nb, 1, 1)
    obs = torch.ones(T, nb, dtype=torch.float64, device="cuda") if mask is None else mask.double()
    for _ in range(its):
        Q = torch.linalg.inv(W).permute(1, 2, 0).float().contiguous()
        r = ctx.lgssm(y, A, B, P, Q, m0, S0, mask=mask, per_chain_model=True)
        e = y.double() - torch.einsum("kd,tdb->tkb", Bd, r["mean"].double())
        R = torch.einsum("tb,tkb,tlb->bkl", obs, e, e) + torch.einsum("tb,kd,tdeb,le->bkl", obs, Bd, r["cov"].double(), Bd)
        W = (nu0 + obs.sum(0))[:, None, None] * torch.linalg.inv(torch.as_tensor(Psi0, device="cuda") + R)
    return W


def bench_vmp_wishart(ctx, peak):
    """Fused Wishart-precision VMP (rxg_lgssm_vmp_wishart_f32) vs the composed path on the same inputs, alternated in one
    run; kernel time from CUDA events around the launch (rxg_set_profiling)."""
    gname, plim = gpu_name_and_power_limit()
    g = torch.Generator(device="cuda").manual_seed(13)
    T, nb, its = 1000, 65536, 10
    for d, masked in ((4, False), (4, True), (2, False)):
        m = d
        mod = notebook_model_f32() if d == 4 else notebook_model_d2_f32()
        y = torch.randn(T, m, nb, device="cuda", generator=g) * 3.3
        mask = (torch.rand(T, nb, device="cuda", generator=g) >= 0.1).to(torch.uint8) if masked else None
        nu0, Psi0, W0 = m + 2.0, 10.0 * np.eye(m), 0.1 * np.eye(m)
        fused = lambda: ctx.lgssm_vmp_wishart(y, mod["A"], mod["B"], mod["P"], mod["m0"], mod["S0"], iterations=its,
                                              w_prior=(nu0, Psi0), init_E_W=W0, mask=mask)
        composed = lambda: _composed_wishart(ctx, y, mod, its, nu0, Psi0, W0, mask)
        call_ms, comp_ms, kern_ms = [], [], []
        for _ in range(3):
            call_ms.append(timed(fused, warm=2, reps=3))
            comp_ms.append(timed(composed, warm=1, reps=2))
            ctx.set_profiling(True)
            fused()
            kern_ms.append(ctx.profile_last_ms()[0])
            ctx.set_profiling(False)
        kms, cms, pms = float(np.median(kern_ms)), float(np.median(call_ms)), float(np.median(comp_ms))
        bf, bc, fl = vmp_wishart_counts(d, m, masked)
        n = T * nb * its
        t_hbm, t_fp32 = bf * n / (peak * 1e9), fl * n / 67e12
        print(json.dumps({"what": "Wishart-precision VMP around the smoother (lgssm_vmp_wishart_kernel)", "d": d, "m": m,
                          "T": T, "batch": nb, "iterations": its, "mask_10pct": masked, "kernel_ms": kms, "call_ms": cms,
                          "ms_per_iteration": kms / its, "composed_path_ms": pms, "speedup_vs_composed": pms / cms,
                          "bytes_per_chain_step_iteration": bf, "composed_bytes_per_chain_step_iteration": bc,
                          "flops_per_chain_step_iteration": fl, "achieved_GBs": bf * n / kms / 1e6,
                          "achieved_TFLOPs": fl * n / kms / 1e9,
                          "bound": "hbm" if t_hbm >= t_fp32 else "fp32",
                          "kernel_frac_of_bound": max(t_hbm, t_fp32) * 1e3 / kms,
                          "peak_hbm_gbs": peak, "peak_fp32_tflops": 67, "gpu": gname, "power_limit": plim}), flush=True)
        del y, mask
        torch.cuda.empty_cache()


def bench_vmp_noise(ctx, peak):
    """Learned process precision (rxg_lgssm_vmp_noise_f32: learn P, learn P and Q) against the learned observation
    precision alone (rxg_lgssm_vmp_wishart_f32), alternated in one run on the same data; kernel time from CUDA events
    around the launch (rxg_set_profiling)."""
    gname, plim = gpu_name_and_power_limit()
    g = torch.Generator(device="cuda").manual_seed(14)
    T, nb, its = 1000, 65536, 10
    for d in (4, 2):
        m = d
        mod = notebook_model_f32() if d == 4 else notebook_model_d2_f32()
        y = torch.randn(T, m, nb, device="cuda", generator=g) * 3.3
        q_prior, q_init = (m + 2.0, 10.0 * np.eye(m)), 0.1 * np.eye(m)
        p_prior, p_init = (d + 2.0, 0.1 * np.eye(d)), np.linalg.inv(np.asarray(mod["P"], np.float64))
        calls = {"Q": lambda: ctx.lgssm_vmp_wishart(y, mod["A"], mod["B"], mod["P"], mod["m0"], mod["S0"], iterations=its,
                                                    w_prior=q_prior, init_E_W=q_init),
                 "P": lambda: ctx.lgssm_vmp_noise(y, mod["A"], mod["B"], mod["m0"], mod["S0"], Q=mod["Q"], p_prior=p_prior,
                                                  p_init=p_init, iterations=its),
                 "PQ": lambda: ctx.lgssm_vmp_noise(y, mod["A"], mod["B"], mod["m0"], mod["S0"], p_prior=p_prior,
                                                   p_init=p_init, q_prior=q_prior, q_init=q_init, iterations=its)}
        kern = {k: [] for k in calls}
        call = {k: [] for k in calls}
        for _ in range(3):
            for k, fn in calls.items():
                call[k].append(timed(fn, warm=2, reps=3))
                ctx.set_profiling(True)
                fn()
                kern[k].append(ctx.profile_last_ms()[0])
                ctx.set_profiling(False)
        for k in calls:
            kms, cms = float(np.median(kern[k])), float(np.median(call[k]))
            bf, _, fl = vmp_wishart_counts(d, m, False, learn=k)
            n = T * nb * its
            t_hbm, t_fp32 = bf * n / (peak * 1e9), fl * n / 67e12
            print(json.dumps({"what": f"noise-precision VMP around the smoother, learn {k} (lgssm_vmp_wishart_kernel)",
                              "learn": k, "d": d, "m": m, "T": T, "batch": nb, "iterations": its, "kernel_ms": kms,
                              "kernel_ms_runs": kern[k], "call_ms": cms, "ms_per_iteration": kms / its,
                              "bytes_per_chain_step_iteration": bf, "flops_per_chain_step_iteration": fl,
                              "achieved_GBs": bf * n / kms / 1e6, "achieved_TFLOPs": fl * n / kms / 1e9,
                              "bound": "hbm" if t_hbm >= t_fp32 else "fp32",
                              "kernel_frac_of_hbm_bound": t_hbm * 1e3 / kms,
                              "kernel_frac_of_bound": max(t_hbm, t_fp32) * 1e3 / kms,
                              "peak_hbm_gbs": peak, "peak_fp32_tflops": 67, "gpu": gname, "power_limit": plim}), flush=True)
        del y
        torch.cuda.empty_cache()


def vmp_transition_counts(d, m, learn):
    """Bytes and FLOPs per (chain, step, iteration) of one non-final iteration of the transition-learning VMP (learn =
    "A", "AP", "APQ"): vmp_wishart_counts of the noise part plus, per step, the tilt exp(-1/2 x' Xi x) (S L, L' S L,
    a d x d Cholesky, Z = S L Ls^-T, the mean and the downdate) and the source-state statistics (X = G Ss (I - A G)' -
    C A', Sxx, Sxr).  The fp64 d^2 x d^2 algebra runs once per iteration, not per step, and is not counted."""
    tri = lambda n: n * (n + 1) // 2
    noise = learn.replace("A", "")
    if noise:
        by, _, fl = vmp_wishart_counts(d, m, False, learn=noise)
    else:       # A alone: y read forward only, plus the stash in both directions
        by = 4 * m + 2 * 4 * (d + tri(d))
        _, _, fl = vmp_wishart_counts(d, m, False, learn="P")
        fl -= 2 * (3 * d ** 3 + 2 * tri(d) * d + d * d + tri(d))      # no R_p pair term
    tilt = d ** 3 + tri(d) * d + d ** 3 // 6 + d ** 3 // 2 + d * d + d * d // 2 + d * d + tri(d) * d
    stats = d ** 3 + d ** 3 + d ** 3 + d ** 3 + d * d + tri(d) + d * d
    return by, fl + 2 * (tilt + stats)


def bench_vmp_transition(ctx, peak):
    """Learned transition matrix (rxg_lgssm_vmp_transition_f32: A alone, A + P, A + P + Q) against the learned noise
    precisions with A known (rxg_lgssm_vmp_noise_f32, learn P + Q), alternated in one run on the same data; kernel time
    from CUDA events around the launch (rxg_set_profiling)."""
    gname, plim = gpu_name_and_power_limit()
    g = torch.Generator(device="cuda").manual_seed(16)
    T, nb, its = 1000, 65536, 10
    for d in (4, 2):
        m = d
        mod = notebook_model_f32() if d == 4 else notebook_model_d2_f32()
        y = torch.randn(T, m, nb, device="cuda", generator=g) * 3.3
        q_prior, q_init = (m + 2.0, 10.0 * np.eye(m)), 0.1 * np.eye(m)
        p_prior, p_init = (d + 2.0, 0.1 * np.eye(d)), np.linalg.inv(np.asarray(mod["P"], np.float64))
        n = d * d
        a_prior = (np.asarray(mod["A"], np.float64).reshape(-1), np.eye(n))
        a_init = (np.asarray(mod["A"], np.float64).reshape(-1), 0.01 * np.eye(n))
        common = dict(a_prior=a_prior, a_init=a_init, iterations=its)
        calls = {"PQ": lambda: ctx.lgssm_vmp_noise(y, mod["A"], mod["B"], mod["m0"], mod["S0"], p_prior=p_prior,
                                                   p_init=p_init, q_prior=q_prior, q_init=q_init, iterations=its),
                 "A": lambda: ctx.lgssm_vmp_transition(y, mod["B"], mod["m0"], mod["S0"], P=mod["P"], Q=mod["Q"], **common),
                 "AP": lambda: ctx.lgssm_vmp_transition(y, mod["B"], mod["m0"], mod["S0"], p_prior=p_prior, p_init=p_init,
                                                        Q=mod["Q"], **common),
                 "APQ": lambda: ctx.lgssm_vmp_transition(y, mod["B"], mod["m0"], mod["S0"], p_prior=p_prior,
                                                         p_init=p_init, q_prior=q_prior, q_init=q_init, **common)}
        kern = {k: [] for k in calls}
        call = {k: [] for k in calls}
        for _ in range(3):
            for k, fn in calls.items():
                call[k].append(timed(fn, warm=2, reps=3))
                ctx.set_profiling(True)
                fn()
                kern[k].append(ctx.profile_last_ms()[0])
                ctx.set_profiling(False)
        for k in calls:
            kms, cms = float(np.median(kern[k])), float(np.median(call[k]))
            if k == "PQ":
                bf, _, fl = vmp_wishart_counts(d, m, False, learn="PQ")
            else:
                bf, fl = vmp_transition_counts(d, m, k)
            nn = T * nb * its
            t_hbm, t_fp32 = bf * nn / (peak * 1e9), fl * nn / 67e12
            print(json.dumps({"what": f"transition-learning VMP around the smoother, learn {k} (lgssm_vmp_wishart_kernel)",
                              "learn": k, "d": d, "m": m, "T": T, "batch": nb, "iterations": its, "kernel_ms": kms,
                              "kernel_ms_runs": kern[k], "call_ms": cms, "ms_per_iteration": kms / its,
                              "bytes_per_chain_step_iteration": bf, "flops_per_chain_step_iteration": fl,
                              "achieved_GBs": bf * nn / kms / 1e6, "achieved_TFLOPs": fl * nn / kms / 1e9,
                              "bound": "hbm" if t_hbm >= t_fp32 else "fp32",
                              "kernel_frac_of_hbm_bound": t_hbm * 1e3 / kms,
                              "kernel_frac_of_bound": max(t_hbm, t_fp32) * 1e3 / kms,
                              "peak_hbm_gbs": peak, "peak_fp32_tflops": 67, "gpu": gname, "power_limit": plim}), flush=True)
        del y
        torch.cuda.empty_cache()


def bench_gmm(ctx, peak):
    """Gaussian-mixture VMP (rxg_gmm_vmp_f32), N = 500 points per data set, 25 iterations, 65 536 data sets, free energy
    on; time from CUDA events around the call (host validation and the constant upload included, both O(K d^3)).  Per
    point, component and iteration the data pass does ~(d + 2 tri(d) + 4) fp32 flops, ~(3 + 2 d + 2 tri(d)) fp64 flops
    and reads the component's constants (4 (d + tri(d) + 1) B) and updates its fp64 accumulators (16 (1 + d + tri(d)) B)
    in shared memory; the bound is the largest of the HBM, fp32, fp64 and shared-memory times."""
    gname, plim = gpu_name_and_power_limit()
    g = torch.Generator(device="cuda").manual_seed(17)
    N, nb, its = 500, 65536, 25
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    smem_tbs = sm * 128 * 1.98e9 / 1e12                          # 128 B / clock / SM at the 1.98 GHz boost clock
    for d, K in ((2, 3), (4, 8)):
        tri = d * (d + 1) // 2
        centres = torch.randn(K, d, device="cuda", generator=g) * 10.0
        lab = torch.randint(0, K, (N, nb), device="cuda", generator=g)
        y = (centres[lab].permute(0, 2, 1) + torch.randn(N, d, nb, device="cuda", generator=g)).contiguous()
        eye = np.tile(np.eye(d), (K, 1, 1))
        args = (np.ones(K), np.zeros((K, d)), 1e4 * eye, np.full(K, d + 1.0), eye, np.ones(K),
                centres.cpu().numpy() + 1.0, 10.0 * eye, np.full(K, d + 1.0), eye)
        runs = [timed(lambda: ctx.gmm_vmp(y, *args, iterations=its), warm=2, reps=3) for _ in range(3)]
        ms = float(np.median(runs))
        n = N * nb * its
        by = 4 * d
        f32_fl, f64_fl = K * (d + 2 * tri + 4), K * (3 + 2 * d + 2 * tri)
        sh = K * (4 * (d + tri + 1) + 16 * (1 + d + tri))
        t = {"hbm": by * n / (peak * 1e9), "fp32": f32_fl * n / 67e12, "fp64": f64_fl * n / 34e12, "shared": sh * n / (smem_tbs * 1e12)}
        bound = max(t, key=t.get)
        print(json.dumps({"what": "Gaussian-mixture VMP (gmm_vmp_kernel), free energy on", "d": d, "K": K, "N": N, "batch": nb,
                          "iterations": its, "ms": ms, "ms_runs": runs, "ms_per_iteration": ms / its,
                          "bytes_per_chain": N * d * 4 * its, "achieved_GBs": by * n / ms / 1e6,
                          "bound": bound, "bound_ms": {k: v * 1e3 for k, v in t.items()}, "frac_of_bound": t[bound] * 1e3 / ms,
                          "peak_hbm_gbs": peak, "peak_fp32_tflops": 67, "peak_fp64_tflops": 34, "shared_tbs": smem_tbs,
                          "gpu": gname, "power_limit": plim}), flush=True)
        del y
        torch.cuda.empty_cache()


def bench_hmm(ctx, peak):
    """Hidden Markov model VMP (rxg_hmm_vmp_f32), T = 1000 steps, 20 iterations, 65 536 chains, A and B learned, free
    energy on; time from CUDA events around the call (host validation and the constant upload included, both O(M K)).
    Algorithmic bytes per (chain, step): (2 + 8 K) per iteration (x read twice, the forward stash written and read once)
    plus 4 K for q(s) written at the end; per step and iteration ~4 K^2 fp32 FMAs (forward, backward, outer product).
    The symbols are uniform (the sweep's cost does not depend on them)."""
    gname, plim = gpu_name_and_power_limit()
    g = torch.Generator(device="cuda").manual_seed(19)
    T, nb, its = 1000, 65536, 20
    for K, M in ((3, 3), (8, 16)):
        x = torch.randint(0, M, (T, nb), device="cuda", generator=g, dtype=torch.uint8)
        rng = np.random.default_rng(K)
        kw = dict(p0=np.full(K, 1.0 / K), A_prior=np.ones((K, K)) + 4 * np.eye(K), A_init=rng.uniform(0.5, 2.0, (K, K)),
                  B_prior=np.ones((M, K)), B_init=rng.uniform(0.5, 2.0, (M, K)))
        runs = [timed(lambda: ctx.hmm_vmp(x, **kw, iterations=its), warm=2, reps=3) for _ in range(3)]
        ms = float(np.median(runs))
        by = ((2 + 8 * K) * its + 4 * K) * T * nb
        fl = 2 * 4 * K * K * its * T * nb
        t = {"hbm": by / (peak * 1e9), "fp32": fl / 67e12}
        bound = max(t, key=t.get)
        print(json.dumps({"what": "hidden Markov model VMP (hmm_vmp_kernel), A and B learned, free energy on", "K": K, "M": M,
                          "T": T, "batch": nb, "iterations": its, "ms": ms, "ms_runs": runs, "ms_per_iteration": ms / its,
                          "bytes_per_chain_step": by / (T * nb), "achieved_GBs": by / ms / 1e6, "bound": bound,
                          "bound_ms": {k: v * 1e3 for k, v in t.items()}, "frac_of_bound": t[bound] * 1e3 / ms,
                          "peak_hbm_gbs": peak, "peak_fp32_tflops": 67, "gpu": gname, "power_limit": plim}), flush=True)
        del x
        torch.cuda.empty_cache()


def bench_hgf_learn(ctx, peak):
    """HGF with learned kappa and omega (rxg_hgf_vmp_learn_f32), T = 1000 steps, 20 iterations, 65 536 chains, free energy
    on; time from CUDA events around the call.  Per (chain, step, iteration): 36 bytes (y read, the old q(x_t+1), q(z_t+1)
    read and the new q(x_t), q(z_t) written).  MUFU operations, an ESTIMATE counted from the source, not from the SASS:
    three GH-31 products of 62 ex2 each (31 for exp(c z + d z^2 / 2), 31 for the weights), 3 expf of B, 3 square roots,
    6 reciprocals (x, the z product and its Gaussian factor, the two fp64 folds' seeds) and, with the free energy, 2 exp,
    4 log and 2 divisions: ~206.  The two folds sum their moments in fp64, ~3 DFMA per node: ~190 DFMA.  The SFU bound takes
    16 MUFU results per clock per SM at the card's maximum SM clock; FP64 at 34 TFLOP/s (data sheet, H100 SXM)."""
    gname, plim = gpu_name_and_power_limit()
    props = torch.cuda.get_device_properties(0)
    sm = props.multi_processor_count
    q = subprocess.run(["nvidia-smi", "--query-gpu=clocks.max.sm", "--format=csv,noheader,nounits"], capture_output=True,
                       text=True).stdout.split()
    clk, clk_src = (float(q[0]) * 1e6, "nvidia-smi") if q else (1980e6, "data sheet boost clock, not read")
    T, nb, its = 1000, 65536, 20
    from oracle.hgf import generate_data
    _, _, y = generate_data(T, 1024, kappa=0.8, omega=-0.5, z_variance=0.01, y_variance=0.2, seed=3)
    y = torch.as_tensor(np.tile(y, (1, nb // 1024)), device="cuda").contiguous()
    runs = [timed(lambda: ctx.hgf_vmp_learn(y, iterations=its), warm=1, reps=2) for _ in range(3)]
    ms = float(np.median(runs))
    n = T * nb * its
    by, mufu, fl, dfma = 36 * n, 206 * n, 3 * 31 * 8 * n, 190 * n
    t = {"hbm": by / (peak * 1e9), "sfu_estimate": mufu / (16 * sm * clk), "fp32": fl / 67e12, "fp64": 2 * dfma / 34e12}
    bound = max(t, key=t.get)
    st = ctx.hgf_vmp_learn(y, iterations=its)["status"]
    print(json.dumps({"what": "HGF with learned kappa, omega (hgf_learn_kernel), free energy on", "T": T, "batch": nb,
                      "iterations": its, "ms": ms, "ms_runs": runs, "ms_per_iteration": ms / its, "bytes_per_chain_step": 36,
                      "achieved_GBs": by / ms / 1e6, "bound": bound, "bound_ms": {k: v * 1e3 for k, v in t.items()},
                      "frac_of_bound": t[bound] * 1e3 / ms, "flagged_chains": int((st != 0).sum()), "peak_hbm_gbs": peak,
                      "sm_count": sm, "max_sm_clock_mhz": clk / 1e6, "clock_source": clk_src, "gpu": gname, "power_limit": plim}), flush=True)
    del y
    torch.cuda.empty_cache()


def bench_hmm_gauss(ctx, peak):
    """Hidden Markov model with Gaussian emissions (rxg_hmm_gauss_vmp_f32), T = 1000 steps, 20 iterations, 65 536 chains,
    A learned, free energy on; time from CUDA events around the call (host validation and the constant upload included).
    Algorithmic bytes per (chain, step): (8 d + 8 K) per iteration (y read twice, the forward stash written and read once)
    plus 4 K for q(s) written at the end.  The fp64 bound: the backward pass adds gamma into K (1 + d + d(d+1)/2) fp64
    shared-memory accumulators per step (2 flops each), at the H100's 33.5 TFLOP/s fp64 (non-tensor) rate."""
    gname, plim = gpu_name_and_power_limit()
    g = torch.Generator(device="cuda").manual_seed(23)
    T, nb, its = 1000, 65536, 20
    for K, d in ((3, 2), (8, 4)):
        y = 3.0 * torch.randn(T, d, nb, device="cuda", generator=g)
        rng = np.random.default_rng(K)
        kw = dict(p0=np.full(K, 1.0 / K), A_prior=np.ones((K, K)) + 4 * np.eye(K), A_init=rng.uniform(0.5, 2.0, (K, K)),
                  mu0=np.zeros((K, d)), V0=np.stack([100.0 * np.eye(d)] * K), nu0=np.full(K, d + 2.0),
                  S0=np.stack([np.eye(d) / (d + 2.0)] * K), m_init=3.0 * rng.standard_normal((K, d)),
                  Vm_init=np.stack([np.eye(d)] * K), nu_init=np.full(K, d + 2.0), S_init=np.stack([np.eye(d) / (d + 2.0)] * K))
        runs = [timed(lambda: ctx.hmm_gauss_vmp(y, **kw, iterations=its), warm=2, reps=3) for _ in range(3)]
        ms = float(np.median(runs))
        by = ((8 * d + 8 * K) * its + 4 * K) * T * nb
        fl64 = 2 * K * (1 + d + d * (d + 1) // 2) * its * T * nb
        t = {"hbm": by / (peak * 1e9), "fp64_accumulators": fl64 / 33.5e12}
        bound = max(t, key=t.get)
        print(json.dumps({"what": "Gaussian-emission HMM VMP (hmm_gauss_vmp_kernel), A learned, free energy on", "K": K,
                          "d": d, "T": T, "batch": nb, "iterations": its, "ms": ms, "ms_runs": runs,
                          "ms_per_iteration": ms / its, "bytes_per_chain_step": by / (T * nb), "achieved_GBs": by / ms / 1e6,
                          "bound": bound, "bound_ms": {k: v * 1e3 for k, v in t.items()}, "frac_of_bound": t[bound] * 1e3 / ms,
                          "peak_hbm_gbs": peak, "gpu": gname, "power_limit": plim}), flush=True)
        del y
        torch.cuda.empty_cache()


def bench_binomial(ctx):
    """Bayesian binomial regression (rxg_binomial_polya_vmp_f32) on both kernels, forced through RXG_OPT_POLYA_PATH
    (1 = one thread per chain, 2 = chain groups), on the same inputs: the reference test's workload (20 chains, N = 1000,
    p = 2, 100 iterations), large batches (65 536 chains, N = 1000, p = 2 and 8, 20 iterations), then a batch x N grid at
    p = 2, 20 iterations, that places the automatic choice.  Free energy on.  Time from CUDA events around the call.
    Algorithmic bytes: every pass reads x, y and n once, (4 p + 8) per sample and chain, over iterations + 1 passes; the
    fraction is of the 3.35 TB/s data-sheet HBM3 bandwidth of the H100 SXM."""
    gname, plim = gpu_name_and_power_limit()
    g = torch.Generator(device="cuda").manual_seed(31)

    def one(what, nb, N, p, its, reps):
        X = torch.randn(N, p, nb, device="cuda", generator=g)
        n = torch.randint(5, 21, (N, nb), device="cuda", generator=g, dtype=torch.int32)
        beta = torch.randn(p, nb, device="cuda", generator=g)
        prob = torch.sigmoid(torch.einsum("ijb,jb->ib", X, beta))
        y = torch.binomial(n.float(), prob).to(torch.int32)
        by = (its + 1) * N * nb * (4 * p + 8)
        row = {"what": what, "batch": nb, "N": N, "p": p, "iterations": its, "algorithmic_bytes": by}
        for path in (1, 2):
            ctx.set_option("polya_path", path)
            f = lambda: ctx.binomial_polya_vmp(X, y, np.zeros(p), np.eye(p), ntrials=n, iterations=its)
            runs = [timed(f, warm=1, reps=reps) for _ in range(3)]
            ms = float(np.median(runs))
            row[f"ms_path{path}"] = ms
            row[f"frac_of_3350GBs_path{path}"] = by / (ms * 1e-3) / 3.35e12
        ctx.set_option("polya_path", 0)
        row.update(gpu=gname, power_limit=plim)
        print(json.dumps(row), flush=True)
        del X, y, n
        torch.cuda.empty_cache()

    one("reference workload", 20, 1000, 2, 100, 5)
    for p in (2, 8):
        one("large batch", 65536, 1000, p, 20, 2)
    for nb in (20, 1024, 4096, 8448, 16384, 65536):
        for N in (100, 1000, 10000):
            one("grid", nb, N, 2, 20, 2)


def bench_multinomial(ctx):
    """Bayesian multinomial regression (rxg_multinomial_polya_vmp_f32 / _online_f32): the reference test's workloads
    (offline: 1 chain, n = 1000, K = 10, 100 iterations; online: 1 chain, T = 5000, K = 40) and large batches (offline
    65 536 chains at K = 10 and 4096 at K = 40, n = 1000, 100 iterations; online 4096 chains, T = 1000, K = 10 and 40, no
    covariance history).  Free energy on.  Call time from CUDA events around the call; per-kernel times from
    torch.profiler in a separate pass.  The data pass reads y once, 4 n K bytes per chain (fraction of the 3.35 TB/s
    data-sheet HBM3 bandwidth of the H100 SXM); a step does D^3 + D^2 fp64 FMAs (D Sherman-Morrison updates of D^2
    entries, then the mean)."""
    from torch.profiler import ProfilerActivity, profile
    gname, plim = gpu_name_and_power_limit()
    g = torch.Generator(device="cuda").manual_seed(41)

    def counts(n, K, nb, N):
        p = torch.softmax(torch.randn(K, nb, device="cuda", generator=g), 0)
        c = torch.distributions.Multinomial(N, probs=p.T).sample((n,))          # [n, nb, K]
        return c.permute(0, 2, 1).contiguous().to(torch.int32)

    def kernel_ms(f):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            f()
            torch.cuda.synchronize()
        out = {}
        for e in prof.key_averages():
            if "mnp_" in e.key:
                name = e.key.split("mnp_")[1].split("_kernel")[0]
                out[name] = out.get(name, 0.0) + e.device_time_total / 1e3
        return out

    def one(what, mode, nb, n, K, N, its, reps):
        D = K - 1
        y = counts(n, K, nb, N)
        xi0, W0 = np.zeros(D), float(K) * np.eye(D)
        if mode == "offline":
            f = lambda: ctx.multinomial_polya_vmp(y, xi0, W0, iterations=its)
            steps = its * nb
        else:
            f = lambda: ctx.multinomial_polya_online(y, xi0, W0, keep_cov=nb == 1)
            steps = n * nb
        ms = float(np.median([timed(f, warm=1, reps=reps) for _ in range(3)]))
        k = kernel_ms(f)
        row = {"what": what, "mode": mode, "batch": nb, "n" if mode == "offline" else "T": n, "K": K, "trials": N,
               "iterations": its, "ms_call": ms, "kernel_ms": k}
        fma = steps * (D ** 3 + D ** 2)
        step_ms = k.get("vmp" if mode == "offline" else "online", float("nan"))
        row["fp64_fma_per_s"] = fma / (step_ms * 1e-3)
        if mode == "offline":
            by = 4 * n * K * nb
            row["data_bytes"] = by
            row["data_frac_of_3350GBs"] = by / (k.get("data", float("nan")) * 1e-3) / 3.35e12
        row.update(gpu=gname, power_limit=plim)
        print(json.dumps(row), flush=True)
        del y
        torch.cuda.empty_cache()

    one("reference workload", "offline", 1, 1000, 10, 20, 100, 5)
    one("large batch", "offline", 65536, 1000, 10, 20, 100, 2)
    one("large batch", "offline", 4096, 1000, 40, 50, 100, 2)
    one("reference workload", "online", 1, 5000, 40, 50, 1, 2)
    one("large batch", "online", 4096, 1000, 10, 20, 1, 2)
    one("large batch", "online", 4096, 1000, 40, 50, 1, 2)


def bench_delta(ctx):
    """Delta node (NVRTC-compiled user functions).  The paper's pendulum (paper/example.jl: Linearization transition,
    Gamma-learned observation precision, 5 VMP iterations per datum, T = 1000) streamed as one chunk, batch 1 and
    65 536, and the d = 4 constant-velocity tracker with a range-bearing g (the whole-series smoother, T = 1000, batch
    65 536), both methods.  The JIT compile is timed on its own, before and outside the timed window (a fresh module
    per line: the source carries a unique comment).  A pendulum window holds one ``delta_filter_chunk`` call: the
    kernel plus the call's host work (argument packing, the history outputs from torch's caching allocator); resetting
    the carry happens before the window.  The paper's published 162 ms (median, one chain, Julia on a CPU)
    is a different machine and a different schedule; the ratio is printed with that caveat."""
    from oracle import delta as D
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from delta_models import PENDULUM_SRC, TRACKER_SRC
    gname, plim = gpu_name_and_power_limit()
    T = 1000
    _, _, obs = D.dataset(T, precision=1.0, seed=42)
    for method, mname in ((0, "Linearization"), (1, "Unscented")):
        t0 = __import__("time").perf_counter()
        mod = ctx.delta_model(PENDULUM_SRC + f"\n// bench {mname}\n", "pendulum", 2, 1, method)
        jit_ms = (__import__("time").perf_counter() - t0) * 1e3
        for nb in (1, 65536):
            y = torch.as_tensor(np.repeat(obs[:, None, None], nb, 2), dtype=torch.float32, device="cuda").contiguous()
            init = [torch.as_tensor(np.repeat(np.asarray(v, np.float32)[..., None], nb, -1), device="cuda").contiguous()
                    for v in ([0.5, 0.0], 0.01 * np.eye(2), [1.0, 0.01])]

            carry = [t.clone() for t in init]

            def run():
                return ctx.delta_filter_chunk(mod, y, np.zeros((2, 2)), *carry[:2], B=np.array([[1.0, 0.0]]),
                                              carry_tau=carry[2], iters=5)

            def timed_stream(reps):
                """Events around the one call: the carry is reset to the initial marginals before, outside the window."""
                ts = []
                for _ in range(reps):
                    for c, i in zip(carry, init):
                        c.copy_(i)
                    torch.cuda.synchronize()
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    run()
                    e1.record()
                    torch.cuda.synchronize()
                    ts.append(e0.elapsed_time(e1))
                return float(np.median(ts))
            timed_stream(2)
            runs = [timed_stream(5) for _ in range(3)]
            ms = float(np.median(runs))
            for c, i in zip(carry, init):
                c.copy_(i)
            st = run()["status"]
            print(json.dumps({"what": f"pendulum stream (paper/example.jl), {mname}, 5 VMP iterations per datum",
                              "T": T, "batch": nb, "ms": ms, "ms_runs": runs, "us_per_chain_datum": ms * 1e3 / (T * nb),
                              "jit_compile_ms": jit_ms, "flagged_chains": int((st != 0).sum()),
                              "paper_reference_ms": 162.086, "paper_reference_note": "Julia RxInfer on a CPU, one chain, "
                              "median; different hardware and a reactive per-datum schedule", "gpu": gname,
                              "power_limit": plim}), flush=True)
            del y, init
    nb = 65536
    P, Q = np.diag([1e-3, 1e-3, 1e-2, 1e-2]), np.diag([0.01, 0.001])
    m0, S0 = np.array([1.0, 2.0, 0.5, -0.3]), np.diag([0.1, 0.1, 0.05, 0.05])
    rng = np.random.default_rng(1)
    y = torch.as_tensor(np.tile(np.stack([np.hypot(4 + 0.05 * np.arange(T), 4.0), np.full(T, 0.7)], 1)[:, :, None],
                                (1, 1, nb)) + rng.normal(0, 0.01, (T, 2, 1)), dtype=torch.float32, device="cuda").contiguous()
    for method, mname in ((0, "Linearization"), (1, "Unscented")):
        t0 = __import__("time").perf_counter()
        mod = ctx.delta_model(TRACKER_SRC + f"\n// bench {mname}\n", "cv", 4, 2, method, g_name="range_bearing")
        jit_ms = (__import__("time").perf_counter() - t0) * 1e3
        runs = [timed(lambda: ctx.delta_smooth(mod, y, m0, S0, P, Q), warm=1, reps=3) for _ in range(3)]
        ms = float(np.median(runs))
        # bytes per (chain, step): y read, filtered mean + cov written, read back and the smoothed pair written
        by = T * nb * 4 * (2 + 3 * (4 + 16))
        st = ctx.delta_smooth(mod, y, m0, S0, P, Q)["status"]
        print(json.dumps({"what": f"range-bearing tracker smoother d = 4, m = 2, {mname}", "T": T, "batch": nb, "ms": ms,
                          "ms_runs": runs, "achieved_GBs": by / ms / 1e6, "jit_compile_ms": jit_ms,
                          "flagged_chains": int((st != 0).sum()), "gpu": gname, "power_limit": plim}), flush=True)
    del y
    torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--which", default="per_chain,filter,hgf,rules,vmp,scaling_T,large,stream,round2")
    args = ap.parse_args()
    which = set(args.which.split(","))
    ctx = rx.Context(0)
    peak, _ = peaks()
    if "predict" in which:
        bench_predict(ctx, peak)
    if "binomial" in which:
        bench_binomial(ctx)
    if "multinomial" in which:
        bench_multinomial(ctx)
    if "inputs" in which:
        bench_inputs(ctx, peak)
    if "vmp_wishart" in which:
        bench_vmp_wishart(ctx, peak)
    if "vmp_noise" in which:
        bench_vmp_noise(ctx, peak)
    if "vmp_transition" in which:
        bench_vmp_transition(ctx, peak)
    if "gmm" in which:
        bench_gmm(ctx, peak)
    if "hmm" in which:
        bench_hmm(ctx, peak)
    if "hgf_learn" in which:
        bench_hgf_learn(ctx, peak)
    if "hmm_gauss" in which:
        bench_hmm_gauss(ctx, peak)
    if "delta" in which:
        bench_delta(ctx)
    mod = notebook_model_f32()
    kw = dict(A=mod["A"], B=mod["B"], P=mod["P"], Q=mod["Q"], m0=mod["m0"], S0=mod["S0"])
    T, batch = 1000, 65536
    g = torch.Generator(device="cuda").manual_seed(7)

    if which & {"per_chain", "filter"}:
        y = torch.randn(T, 4, batch, device="cuda", generator=g) * 3.3
        mean = torch.empty(T, 4, batch, device="cuda"); cov = torch.empty(T, 4, 4, batch, device="cuda")
        if "per_chain" in which:
            ms = timed(lambda: ctx.lgssm(y, **kw, smooth=True, out_mean=mean, out_cov=cov, force_per_chain_path=True))
            print(json.dumps({"what": "lgssm smooth, per-chain covariance recursion (lgssm_chain_kernel)", "d": 4, "T": T,
                              "batch": batch, "ms": ms, "messages_per_s": 6 * T * batch / ms * 1e3,
                              "algorithmic_GBs": 96 * T * batch / ms / 1e6, "frac_of_hbm_peak": 96 * T * batch / ms / 1e6 / peak}))
        if "filter" in which:
            for tf in (False, True):
                ms = timed(lambda: ctx.lgssm(y, **kw, smooth=False, out_mean=mean, out_cov=cov, transition_first=tf))
                print(json.dumps({"what": "lgssm filter (forward half), gain-table path", "transition_first": tf, "d": 4, "T": T,
                                  "batch": batch, "ms": ms, "messages_per_s": 4 * T * batch / ms * 1e3,
                                  "algorithmic_GBs": 96 * T * batch / ms / 1e6}))
        del y, mean, cov

    if "scaling_T" in which:
        # the notebook's scaling table (ipynb:795-806) at d = 2, batched: T from 50 to 50 000
        m2 = notebook_model_d2_f32()
        for TT in (50, 1000, 10000, 50000):
            b = max(1024, min(65536, (1 << 26) // TT))
            y = torch.randn(TT, 2, b, device="cuda", generator=g) * 3.3
            ms = timed(lambda: ctx.lgssm(y, **m2, smooth=True), warm=3, reps=3)
            print(json.dumps({"what": "lgssm smooth d=2 (notebook scaling table shape)", "T": TT, "batch": b, "ms": ms,
                              "messages_per_s": 6 * TT * b / ms * 1e3, "ms_per_chain_equiv": ms / b}))
            del y

    if "stream" in which:
        # what HBM delivers to a dependency-free streaming kernel for a given read : write mix (the headline cluster sweep
        # reads y once and writes means and covariances: 1.05 GB in and 5.24 GB out per launch, i.e. ~1 : 5; the lock-step
        # kernel's checkpoint variant moves ~2 : 5)
        n = 1 << 28                                            # 1 GiB per row: far beyond L2
        for nr, nw in ((1, 1), (1, 5), (2, 5), (0, 4), (4, 1)):
            src = torch.randn(max(nr, 1), n, device="cuda")[:nr] if nr else torch.empty(0, n, device="cuda")
            dst = torch.empty(nw, n, device="cuda")
            ms = timed(lambda: ctx.selftest_stream(src, dst), warm=3, reps=5)
            print(json.dumps({"what": "stream_mix_kernel (HBM yardstick)", "rows_read": nr, "rows_written": nw, "ms": ms,
                              "GBs": (nr + nw) * n * 4 / ms / 1e6, "frac_of_copy_peak": (nr + nw) * n * 4 / ms / 1e6 / peak}))
            del src, dst

    if "round2" in which:
        # round-2 additions: shared vs per-chain missing-data pattern, embedded shapes, the generic one-CTA-per-chain kernel,
        # the IID Wishart VMP
        y = torch.randn(T, 4, batch, device="cuda", generator=g) * 3.3
        mean = torch.empty(T, 4, batch, device="cuda"); cov = torch.empty(T, 4, 4, batch, device="cuda")
        tm = (np.random.default_rng(1).random(T) > 0.2).astype(np.uint8)
        full = torch.as_tensor(np.repeat(tm[:, None], batch, axis=1), device="cuda")
        for name, mk in (("shared pattern, RXG_MASK_SHARED (gain-table path)", tm), ("same pattern as a per-chain mask (per-chain covariance recursion)", full)):
            ms = timed(lambda: ctx.lgssm(y, **kw, smooth=True, out_mean=mean, out_cov=cov, mask=mk))
            print(json.dumps({"what": "lgssm smooth with 20 % missing steps: " + name, "d": 4, "T": T, "batch": batch, "ms": ms,
                              "messages_per_s": 6 * T * batch / ms * 1e3, "frac_of_hbm_peak": 96 * T * batch / ms / 1e6 / peak}))
        del y, mean, cov, full
        rng = np.random.default_rng(5)
        for d, m, b in ((5, 3, 65536), (6, 6, 65536), (12, 7, 16384), (16, 16, 16384)):
            Aq, _ = np.linalg.qr(rng.standard_normal((d, d)))
            md = {k: v.astype(np.float32) for k, v in dict(A=0.95 * Aq, B=rng.standard_normal((m, d)) / np.sqrt(d), P=0.2 * np.eye(d),
                                                          Q=1.5 * np.eye(m), m0=np.zeros(d), S0=5.0 * np.eye(d)).items()}
            y = torch.randn(T, m, b, device="cuda", generator=g)
            mean = torch.empty(T, d, b, device="cuda"); cov = torch.empty(T, d, d, b, device="cuda")
            ms = timed(lambda: ctx.lgssm(y, **md, smooth=True, out_mean=mean, out_cov=cov), warm=2, reps=3)
            print(json.dumps({"what": "lgssm smooth, shared model, general shape" + (" (native)" if (d, m) in ((6, 6), (16, 16)) else " (embedded in the next native shape)"),
                              "d": d, "m": m, "T": T, "batch": b, "ms": ms, "messages_per_s": 6 * T * b / ms * 1e3,
                              "algorithmic_GBs": 4 * (m + d + d * d) * T * b / ms / 1e6}))
            del y, mean, cov
        for d, b in ((16, 2048), (64, 512)):
            md = dense_model_f32(d)
            y = torch.randn(T, d, b, device="cuda", generator=g) * 3.3
            mk = (torch.rand(T, b, device="cuda", generator=g) > 0.2).to(torch.uint8)
            mean = torch.empty(T, d, b, device="cuda"); cov = torch.empty(T, d, d, b, device="cuda")
            ms = timed(lambda: ctx.lgssm(y, **md, smooth=True, out_mean=mean, out_cov=cov, mask=mk), warm=1, reps=2)
            print(json.dumps({"what": "lgssm smooth, per-chain missing data, generic one-CTA-per-chain kernel (CUDA cores)", "d": d, "T": T,
                              "batch": b, "ms": ms, "messages_per_s": 6 * T * b / ms * 1e3, "us_per_chain_step": ms * 1e3 / (T * b) * min(b, 132 * (2 if d <= 32 else 1))}))
            del y, mk, mean, cov
        yw = torch.randn(1500, 2, 32768, device="cuda", generator=g)
        ms = timed(lambda: ctx.mv_iid_wishart_vmp(yw, iterations=10), warm=2, reps=3)
        print(json.dumps({"what": "IID Wishart-precision VMP (mv_iid_precision model), 10 iterations", "d": 2, "N": 1500, "batch": 32768, "ms": ms,
                          "datasets_per_s": 32768 / ms * 1e3, "GBs": yw.numel() * 4 / ms / 1e6}))
        del yw
        # latent AR (lar_tests.jl model): T = 500, 15 structured-VMP iterations = 15 filter + RTS passes per series
        for order, bl in ((1, 65536), (5, 16384)):
            yl = torch.randn(500, bl, device="cuda", generator=g)
            ms = timed(lambda: ctx.lar_vmp(yl, order, 5.0, iterations=15), warm=1, reps=3)
            print(json.dumps({"what": "latent AR structured VMP (lar_tests.jl model), 15 iterations", "order": order, "T": 500, "batch": bl,
                              "ms": ms, "series_per_s": bl / ms * 1e3, "chain_steps_per_s": 2 * 15 * 500 * bl / ms * 1e3}))
            del yl

    if "large" in which:
        # BASELINE configs[2] (d = 64, T = 1000, batch = 4096) and the smaller tensor-core sizes; shared model.
        # flops: textbook Kalman + RTS mean recursions only = 2 * (2 d^2 [F x + K y] + 2 d^2 [E x + G x]) per (chain, step)
        ctx.set_profiling(True)
        for d, b in ((64, 4096), (64, 18944), (32, 16384), (16, 65536)):
            md = dense_model_f32(d)
            y = torch.randn(T, d, b, device="cuda", generator=g) * 3.3
            mean = torch.empty(T, d, b, device="cuda")
            for no_umma in ("0", "1"):
                ctx.set_option("no_umma", int(no_umma))
                sw, gn = [], []
                def run():
                    ctx.lgssm(y, **md, smooth=True, out_mean=mean, cov_shared_out=True)
                    a, bb = ctx.profile_last_ms(); sw.append(a); gn.append(bb)
                ms = timed(run, warm=2, reps=3)
                print(json.dumps({"what": "lgssm smooth, large-state family (shared model, cov de-duplicated)", "d": d, "T": T, "batch": b,
                                  "sweep": "wgmma 3xTF32 (umma_ky + lgssm_umma_sweep)" if no_umma == "0" else "FP32 pipe (lgssm_block_sweep)",
                                  "ms": ms, "sweep_ms": float(np.mean(sw[-3:])), "gain_tables_ms": float(np.mean(gn[-3:])),
                                  "messages_per_s": 6 * T * b / ms * 1e3,
                                  "sweep_TFLOPs": 8 * d * d * T * b / (float(np.mean(sw[-3:])) * 1e-3) / 1e12}))
            ctx.set_option("no_umma", 0)
            del y, mean
        ctx.set_profiling(False)

    if "hgf" in which:
        Th, bh, iters = 1000, 32768, 20
        yh = torch.randn(Th, bh, device="cuda", generator=g).cumsum(0) * 0.5
        out = torch.empty(Th, 4, bh, device="cuda")
        ms = timed(lambda: ctx.hgf_filter(yh, iters=iters, out=out), warm=3, reps=3)
        n_exp = (31 + 1 + iters * 32) * Th * bh
        print(json.dumps({"what": "HGF filter (BASELINE configs[3]): GCV node, GH-31, 20 VMP iterations", "T": Th, "batch": bh,
                          "iters": iters, "ms": ms, "vmp_iterations_per_s": iters * Th * bh / ms * 1e3,
                          "messages_per_s": 6 * iters * Th * bh / ms * 1e3, "exp_per_s": n_exp / ms * 1e3,
                          "io_GBs": 20 * Th * bh / ms / 1e6}))

    if "vmp" in which:
        yv = torch.randn(1000, 65536, device="cuda", generator=g).cumsum(0)
        ms = timed(lambda: ctx.lgssm_vmp_gamma(yv, iterations=10), warm=2, reps=3)
        print(json.dumps({"what": "Gamma-precision VMP around scalar smoother, 10 iterations", "T": 1000, "batch": 65536, "ms": ms,
                          "sweeps_per_s": 10 / ms * 1e3}))

    if "rules" in which:
      for n, d in ((1 << 22, 4), (1 << 16, 16), (1 << 14, 64)):       # d = 16 / 64: csrc/rxg_rules_large.cu (configs[2] message size)
        mu = torch.randn(d, n, device="cuda", generator=g)
        X = torch.randn(d, d, n, device="cuda", generator=g)
        S = torch.einsum("ikn,jkn->ijn", X, X).contiguous() + d * torch.eye(d, device="cuda")[:, :, None]
        S = S.contiguous()
        del X
        A = np.asarray(mod["A"]) if d == 4 else np.asarray(dense_model_f32(d)["A"])
        Pm = np.asarray(mod["P"]) if d == 4 else np.eye(d, dtype=np.float32)
        rows = []
        rows.append(("MvNormalMeanCovariance(:out)  (mu, S + Sigma)", timed(lambda: ctx.rule_add_cov(mu, S, Pm)), 2 * (d + d * d) * 4))
        rows.append(("*(:out)  (A mu, A S A')", timed(lambda: ctx.rule_mul_out(A, mu, S)), 2 * (d + d * d) * 4))
        rows.append(("*(:in)   cholinv + A' W A", timed(lambda: ctx.rule_mul_in(A, mu, S)), 2 * (d + d * d) * 4 + 4))
        mu2, S2 = (mu * 0.5).contiguous(), (S * 2.0).contiguous()          # distinct operands: 2 reads + 1 write per message
        rows.append(("prod (xi1 + xi2, W1 + W2)", timed(lambda: ctx.prod_gaussian(mu, S, mu2, S2)), 3 * (d + d * d) * 4))
        rows.append(("mean_cov <-> weightedmean_precision (cholinv)", timed(lambda: ctx.meancov_to_wmp(mu, S)), 2 * (d + d * d) * 4 + 4))
        for name, ms, bytes_per in rows:
            # note: torch.empty_like allocations are inside the timed call (caching allocator)
            print(json.dumps({"what": "rule kernel: " + name, "n": n, "d": d, "ms": ms, "messages_per_s": n / ms * 1e3,
                              "GBs": bytes_per * n / ms / 1e6, "frac_of_hbm_peak": bytes_per * n / ms / 1e6 / peak}))


if __name__ == "__main__":
    main()
