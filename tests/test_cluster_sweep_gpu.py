"""The cluster sweep (`lgssm_cluster_sweep_kernel`, csrc/rxg_lgssm_cluster.cuh), chain by chain, against the fp64 Kalman
filter + RTS smoother of test_shared_sweep_variants.py, and its selection.

The plain smoothing call (no evidence, offset or inputs) at d = m in {1, 2, 3, 4} with whole 32-chain tiles of aligned
buffers and the default dispatch options runs the cluster sweep: one 8-CTA cluster per tile, each CTA a time slice of
8 x 16-step sub-segments, carries scanned through shared and distributed shared memory.  The T below put the last step
on, just before and just after sub-segment and slice edges.  Every other call must keep `lgssm_shared_kernel`; the
launch counter tells the two apart (the cluster sweep launches its per-call scan tables and the sweep, one launch more
than the lock-step kernel)."""
import numpy as np
import pytest
import torch

from oracle import lgssm
from test_shared_sweep_variants import (_kw, covariance_side, gate_cov, gate_mean, offset, pattern, random_model,
                                        reference_sweep, simulate)
from util import f32_model

pytestmark = pytest.mark.gpu

SERVED = [(1, 1), (2, 2), (3, 3), (4, 4)]
EDGE_T = [1, 2, 15, 16, 17, 124, 125, 126, 127, 128, 129, 999, 1000]


def max_T(d, m):
    """Largest T whose CTA (y slice + F, K, E, G records + scan scratch) fits the opt-in shared memory of the device;
    ClusterTab::smem_bytes restated."""
    pad4 = lambda n: (n + 3) // 4 * 4
    fk, eg, rec = pad4(d * d) + pad4(d * m), 2 * pad4(d * d), 2 * pad4(d * d)
    cap = torch.cuda.get_device_properties(0).shared_memory_per_block_optin
    smem = lambda spc: 4 * (spc * 16 * (m * 32 + fk + eg) + (spc + 8) * rec + spc * d * 32 + 2 * d * 32)
    spc = 1
    while smem(spc + 1) <= cap:
        spc += 1
    return spc * 8 * 16


def _launches(ctx, fn):
    l0 = ctx.launches
    r = fn()
    torch.cuda.synchronize()
    return r, ctx.launches - l0


def _smooth(ctx, y, mod, **kw):
    return _launches(ctx, lambda: ctx.lgssm(y, **_kw(mod), smooth=True, **kw))


def _lockstep(ctx, y, mod, **kw):
    ctx.set_option("force_cpt", 2)
    try:
        return _smooth(ctx, y, mod, **kw)
    finally:
        ctx.set_option("force_cpt", 0)


@pytest.mark.parametrize("tf", [False, True])
@pytest.mark.parametrize("d,m", SERVED)
def test_every_chain_against_fp64_reference(ctx, d, m, tf):
    """T over sub-segment (16) and slice (128 at T <= 1024) edges up to the largest T the shared memory holds, prior on
    x[1] or one transition earlier, a shared missing-data pattern at one T; 64 chains (two clusters)."""
    mod = random_model(d, m, seed=8000 + 16 * d + m)
    nb = 64
    for T in EDGE_T + [max_T(d, m)]:
        y = torch.as_tensor(simulate(mod, T, nb, seed=5 * T + d), device="cuda")
        case = f"d={d} m={m} T={T} tf={int(tf)}"
        ref = reference_sweep(mod, y.cpu(), transition_first=tf)
        r, n = _smooth(ctx, y, mod, transition_first=tf)
        _, n_ls = _lockstep(ctx, y, mod, transition_first=tf)
        assert n == n_ls + 1, f"{case}: the cluster sweep did not run ({n} launches, lock-step {n_ls})"
        gate_mean("cluster", case, r["mean"], ref["mean"])
        gate_cov("cluster", case, r["cov"], ref["cov"])
    T = 300
    tm = pattern(T)
    y = torch.as_tensor(simulate(mod, T, nb, seed=d), device="cuda")
    y[torch.as_tensor(tm == 0).cuda()] = 1.0e3                    # values at missing steps must not reach any output
    ref = reference_sweep(mod, y.cpu(), transition_first=tf, cs=covariance_side(mod, T, tm, tf))
    r, _ = _smooth(ctx, y, mod, transition_first=tf, mask=tm)
    gate_mean("cluster", f"d={d} m={m} T={T} tf={int(tf)} shared mask", r["mean"], ref["mean"])


@pytest.mark.parametrize("d,m", SERVED)
def test_beyond_shared_memory_falls_back(ctx, d, m):
    """One slice more than the shared memory holds: the lock-step kernel runs, and is still exact."""
    mod = random_model(d, m, seed=8100 + d)
    T = max_T(d, m) + 8 * 16
    y = torch.as_tensor(simulate(mod, T, 32, seed=d), device="cuda")
    r, n = _smooth(ctx, y, mod)
    _, n_ls = _lockstep(ctx, y, mod)
    assert n == n_ls
    gate_mean("cluster fallback", f"d={d} m={m} T={T}", r["mean"], reference_sweep(mod, y.cpu())["mean"])


def test_more_tiles_than_resident_clusters_and_outputs(ctx):
    """8 192 tiles (far more than the clusters resident at once), per-chain and de-duplicated covariance outputs, no
    covariance output; chain reversal is bit for bit."""
    mod = f32_model(lgssm.notebook_model(4))
    T, nb = 257, 262144
    g = torch.Generator(device="cuda").manual_seed(7)
    y = torch.randn(T, 4, nb, device="cuda", generator=g) * 3.3
    idx = torch.cat([torch.arange(0, 64), torch.arange(nb // 2 - 32, nb // 2 + 32), torch.arange(nb - 64, nb)]).cuda()
    ref = reference_sweep(mod, y[..., idx].contiguous())
    r, n = _smooth(ctx, y, mod)
    gate_mean("cluster tiles", "per-chain cov", r["mean"][..., idx], ref["mean"])
    gate_cov("cluster tiles", "per-chain cov", r["cov"][..., idx], ref["cov"])
    assert torch.equal(r["cov"][..., 0], r["cov"][..., nb - 1])
    cov_tab = r["cov"][..., 0].clone()
    mean = r["mean"]
    del r
    rs, ns = _smooth(ctx, y, mod, cov_shared_out=True)
    assert ns == n and torch.equal(rs["mean"], mean) and torch.equal(rs["cov"], cov_tab)
    del rs
    rn, _ = _smooth(ctx, y, mod, want_cov=False)
    assert rn["cov"] is None and torch.equal(rn["mean"], mean)
    del rn
    rr, _ = _smooth(ctx, y.flip(-1).contiguous(), mod, want_cov=False)
    assert torch.equal(rr["mean"].flip(-1), mean)


def test_full_size_matches_lockstep_kernel(ctx):
    """bench.py's call (notebook model, d = m = 4, T = 1000, 65 536 chains): the cluster sweep against the lock-step
    checkpoint kernel (force_cpt = 2) and against the fp64 reference, every chain; covariances bit for bit."""
    mod = f32_model(lgssm.notebook_model(4))
    g = torch.Generator(device="cuda").manual_seed(4242)
    y = torch.randn(1000, 4, 65536, device="cuda", generator=g) * 3.3
    r, n = _smooth(ctx, y, mod)
    ls, n_ls = _lockstep(ctx, y, mod)
    assert n == n_ls + 1
    assert torch.equal(r["cov"], ls["cov"])
    gate_mean("full", "cluster vs lock-step", r["mean"], ls["mean"])
    ref = reference_sweep(mod, y)
    em = gate_mean("full", "cluster vs fp64", r["mean"], ref["mean"])
    el = gate_mean("full", "lock-step vs fp64", ls["mean"], ref["mean"])
    print(f"full size: worst chain mean rel L2 cluster {em:.2e}, lock-step {el:.2e}")


@pytest.mark.parametrize("what", ["evidence", "offset", "inputs", "filter", "m_below_d", "ragged_batch", "misaligned",
                                  "force_cpt", "sweep_variant", "per_chain_prior"])
def test_calls_outside_the_eligibility_set_keep_the_lockstep_kernel(ctx, what):
    d, m = {"m_below_d": (4, 2)}.get(what, (4, 4))
    mod = random_model(d, m, seed=8200 + d + m)
    T, nb = 40, 64 if what != "ragged_batch" else 70
    y = torch.as_tensor(simulate(mod, T, nb, seed=3), device="cuda")
    u = offset(d, 5)
    kw = {}
    if what == "evidence":
        kw = dict(want_evidence=True)
    elif what == "offset":
        kw = dict(u=u)
    elif what == "inputs":
        kw = dict(inputs=np.tile(u, (T, 1)))
    elif what == "misaligned":
        ym = torch.empty(T * m * nb + 1, device="cuda")[1:].view(T, m, nb)
        y = ym.copy_(y)
    if what == "filter":
        run = lambda: ctx.lgssm(y, **_kw(mod), smooth=False)
    elif what == "per_chain_prior":
        prev = torch.zeros(d, nb, device="cuda")
        run = lambda: ctx.lgssm_filter_chunk(y, mod["A"], mod["B"], mod["P"], mod["Q"], prev, np.eye(d, dtype=np.float32))
    else:
        run = lambda: ctx.lgssm(y, **_kw(mod), smooth=True, **kw)
    if what == "force_cpt":
        ctx.set_option("force_cpt", 2)
    if what == "sweep_variant":
        ctx.set_option("sweep_variant", 1)
    _, n = _launches(ctx, run)
    ctx.set_option("force_cpt", 1)
    ctx.set_option("sweep_variant", 0)
    _, n_ls = _launches(ctx, run)                     # CPT = 1 is never the cluster sweep
    ctx.set_option("force_cpt", 0)
    assert n == n_ls, f"{what}: {n} launches, lock-step {n_ls}"
