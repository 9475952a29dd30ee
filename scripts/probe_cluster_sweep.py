#!/usr/bin/env python
"""Where the headline cluster sweep's time goes: the per-chain covariance stream against what HBM delivers.

bench.py's call (notebook model, d = m = 4, T = 1000, 65 536 chains) runs lgssm_cluster_sweep_kernel, which moves 96 B
per (chain, step): y in (16 B), smoothed means (16 B) and per-chain covariances (64 B) out.  The covariances are 4.19 GB
of the 6.29 GB.  This probe times, alternating, in one process:

  full        profile_last_ms()[0] of bench's exact call (per-chain covariances)
  means_only  the same call with want_cov=False (the sweep with write_cov = 0: y in, means out, 2.1 GB)
  stream      ctx.selftest_stream at the read : write mixes (1, 5) (the sweep's own ~1.05 : 5.24 GB), (0, 4) (pure
              streaming writes) and (1, 1)

and derives the covariance stream's cost (full - means_only), its effective write rate against the (0, 4) rate, and the
whole-kernel floor 6.29 GB / (1, 5) rate.  One JSON line per measurement and a summary line go to stdout and to
OUT/probe_cluster_sweep.jsonl.  RXG_LIB selects the library build, as everywhere in the package.

  python scripts/probe_cluster_sweep.py --out DIR [--reps 5] [--calls 20]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bench import ALGO_BYTES_PER_STEP, BATCH, D, M, T, notebook_model_f32  # noqa: E402


def gpu_info():
    """Card, power limit and SM clocks, read-only."""
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"],
                         capture_output=True, text=True, timeout=30).stdout.strip()
    return dict(zip(q.split(","), (x.strip() for x in out.split(","))))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True, help="directory for probe_cluster_sweep.jsonl")
    ap.add_argument("--reps", type=int, default=5, help="alternations of the three measurements")
    ap.add_argument("--calls", type=int, default=20, help="sweep calls per kernel-time sample")
    args = ap.parse_args()

    import torch
    import rxinfer_jl_b200 as rx

    if not torch.cuda.is_available():
        raise SystemExit("probe_cluster_sweep.py needs a GPU")
    os.makedirs(args.out, exist_ok=True)
    log = open(os.path.join(args.out, "probe_cluster_sweep.jsonl"), "a")

    def emit(obj):
        s = json.dumps(obj)
        print(s, flush=True)
        log.write(s + "\n")

    dev = torch.device("cuda", 0)
    ctx = rx.Context(0)
    mod = notebook_model_f32()
    kw = dict(A=mod["A"], B=mod["B"], P=mod["P"], Q=mod["Q"], m0=mod["m0"], S0=mod["S0"])
    g = torch.Generator(device=dev).manual_seed(42)
    y = torch.randn(T, M, BATCH, device=dev, generator=g) * 3.3
    mean = torch.empty(T, D, BATCH, device=dev)
    cov = torch.empty(T, D, D, BATCH, device=dev)
    ctx.set_profiling(True)

    def sweep_ms(want_cov):
        call = lambda: ctx.lgssm(y, **kw, smooth=True, out_mean=mean, out_cov=cov if want_cov else None,
                                 want_cov=want_cov, asynchronous=True)
        for _ in range(3):
            call()
        ms = []
        for _ in range(args.calls):
            call()
            ms.append(ctx.profile_last_ms()[0])
        return float(np.mean(ms))

    n = 1 << 28                                              # 1 GiB per row: far beyond L2
    mixes = ((1, 5), (0, 4), (1, 1))
    bufs = {}
    for nr, nw in mixes:
        bufs[nr, nw] = (torch.randn(nr, n, device=dev) if nr else torch.empty(0, n, device=dev),
                        torch.empty(nw, n, device=dev))

    def stream_gbs(nr, nw):
        src, dst = bufs[nr, nw]
        for _ in range(3):
            ctx.selftest_stream(src, dst)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(5):
            ctx.selftest_stream(src, dst)
        e1.record()
        torch.cuda.synchronize()
        return (nr + nw) * n * 4 / (e0.elapsed_time(e1) / 5) / 1e6

    info = gpu_info()
    emit({"what": "gpu", **info, "lib": os.path.basename(rx._lib.LIB_PATH)})
    full, means_only, rates = [], [], {m: [] for m in mixes}
    for rep in range(args.reps):
        full.append(sweep_ms(True))
        means_only.append(sweep_ms(False))
        for m in mixes:
            rates[m].append(stream_gbs(*m))
        emit({"what": "rep", "rep": rep, "full_ms": full[-1], "means_only_ms": means_only[-1],
              **{f"stream_{a}_{b}_GBs": rates[a, b][-1] for a, b in mixes}})

    total_bytes = ALGO_BYTES_PER_STEP * T * BATCH
    cov_bytes = 4 * D * D * T * BATCH
    f, mo = float(np.median(full)), float(np.median(means_only))
    r15, r04, r11 = (float(np.median(rates[m])) for m in mixes)
    cov_ms = f - mo
    cov_gbs = cov_bytes / (cov_ms * 1e-3) / 1e9
    emit({"what": "summary", **info, "reps": args.reps, "calls": args.calls,
          "full_ms": {"median": f, "min": min(full), "max": max(full)},
          "means_only_ms": {"median": mo, "min": min(means_only), "max": max(means_only)},
          "stream_GBs": {f"{a}:{b}": float(np.median(rates[a, b])) for a, b in mixes},
          "cov_bytes": cov_bytes, "cov_ms": cov_ms, "cov_GBs": cov_gbs, "cov_frac_of_0_4_rate": cov_gbs / r04,
          "total_bytes": total_bytes, "full_GBs": total_bytes / (f * 1e-3) / 1e9,
          "floor_ms_at_1_5_rate": total_bytes / (r15 * 1e9) * 1e3, "full_over_floor": f / (total_bytes / (r15 * 1e9) * 1e3)})
    log.close()


if __name__ == "__main__":
    main()
