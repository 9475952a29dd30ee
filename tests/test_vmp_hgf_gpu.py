"""GPU parity of the variational members of the path: fused HGF filter (GCV node, GH-31), the Gamma-precision VMP
around a scalar smoother and the streaming mean-field Gamma model.  HGF: the oracle is pinned by the
reference test on its own data stream, free energy included (tests/test_reference_rng_goldens.py, oracle/hgf.py)."""
import os

import numpy as np
import pytest
import torch

from oracle import hgf, vmp
from util import rel_l2

pytestmark = pytest.mark.gpu
# GPU (fp32) vs oracle (fp64) bounds, relative L2 over all (t, chain) -- all inside the contract's 1e-5 (psi / det of the
# GCV joint are in cancellation-free closed form).
# Round 1 needed 1e-4 / 2e-3 / 5e-3 / 5e-3.
HGF_TOL = {"m_x": 1e-6, "v_x": 2e-6, "m_z": 5e-6, "v_z": 5e-6}
GOLD = os.path.join(os.path.dirname(__file__), "golden")


def dev(a):
    return torch.as_tensor(np.ascontiguousarray(a), dtype=torch.float32, device="cuda")


def test_hgf_golden_fixture(ctx):
    z = np.load(os.path.join(GOLD, "hgf_T40_b8.npz"))
    out = ctx.hgf_filter(dev(z["y"]), iters=10).cpu().numpy()
    ref = z["out"]
    for k, tol in ((0, 1e-5), (1, 1e-5), (2, 1e-5), (3, 1e-5)):
        assert rel_l2(out[:, k], ref[:, k]) < tol, k


@pytest.mark.parametrize("iters", [1, 20])
def test_hgf_vs_oracle(ctx, iters):
    _, x, y = hgf.generate_data(300, 130, seed=5)
    ref = hgf.hgf_filter(y, iters=iters)
    out = ctx.hgf_filter(dev(y), iters=iters).cpu().numpy()
    errs = [rel_l2(out[:, k], ref[:, k]) for k in range(4)]
    print("hgf vs oracle relL2 (m_x, v_x, m_z, v_z):", errs, "max abs m_z", np.abs(out[:, 2] - ref[:, 2]).max())
    assert errs[0] < HGF_TOL["m_x"] and errs[1] < HGF_TOL["v_x"] and errs[2] < HGF_TOL["m_z"] and errs[3] < HGF_TOL["v_z"]
    assert np.all(out[:, 1] > 0) and np.all(out[:, 3] > 0)      # hgf_tests.jl:131-132
    inside = np.abs(out[:, 0] - x) < 3 * np.sqrt(out[:, 1])
    assert inside.mean() > 0.95                                  # hgf_tests.jl:127-130


def test_hgf_infer_entry(rx, ctx):
    _, _, y = hgf.generate_data(50, 64, seed=6)
    res = rx.infer(model=rx.hgf(), data={"y": dev(y)}, iterations=10, context=ctx)
    ref = hgf.hgf_filter(y, iters=10)
    assert rel_l2(res.history["xt"].mean().cpu().numpy(), ref[:, 0]) < 1e-6
    # free_energy=True: free_energy_history semantics (per iteration, averaged over the data), vs the oracle's
    resf = rx.infer(model=rx.hgf(), data={"y": dev(y)}, iterations=10, free_energy=True, context=ctx)
    _, fe = hgf.hgf_filter(y, iters=10, return_free_energy=True)
    got = resf.free_energy.cpu().numpy()
    assert got.shape == (10, 64)
    assert np.abs(got - fe.mean(axis=0)).max() < 1e-4


def test_hgf_free_energy_vs_oracle_and_chunks(ctx):
    """Device-side Bethe free energy per (datum, iteration, chain) against the oracle's in-loop value; a stream cut
    into chunks (streaming engine) gives bitwise the single call, free energy included."""
    _, _, y = hgf.generate_data(120, 96, seed=9)
    ref, fe_ref = hgf.hgf_filter(y, iters=8, return_free_energy=True)
    out, fe = ctx.hgf_filter(dev(y), iters=8, want_free_energy=True)
    fe = fe.cpu().numpy()
    assert fe.shape == (120, 8, 96)
    err = np.abs(fe - fe_ref)
    print("hgf free energy: max abs err", err.max(), "mean abs err", err.mean(), "scale", np.abs(fe_ref).mean())
    assert err.max() < 2e-4 and err.mean() < 1e-5
    plain = ctx.hgf_filter(dev(y), iters=8)
    assert torch.equal(plain, out)                              # the FE variant does not perturb the posteriors
    o1, f1 = ctx.hgf_filter(dev(y[:50]), iters=8, want_free_energy=True)
    o2, f2 = ctx.hgf_filter_chunk(dev(y[50:]), o1[-1].contiguous(), iters=8, want_free_energy=True)
    assert torch.equal(torch.cat([o1, o2]), out) and torch.equal(torch.cat([f1, f2]).cpu(), torch.as_tensor(fe))


def test_hgf_full_size_parity_report(ctx):
    """BASELINE configs[3] at its real size (T = 1000, batch = 32 768, 20 VMP iterations): sampled chains against
    the fp64 oracle.  Prints the achieved error per output (the figures DESIGN.md quotes) and holds them to the
    bounds fp32 can honestly keep over a 1000-step recursive filter with 20 fixed-point iterations per step."""
    T, batch, iters = 1000, 32768, 20
    idx = np.arange(0, batch, batch // 48)[:48]
    _, _, ys = hgf.generate_data(T, 48, seed=21)
    g = torch.Generator(device="cuda").manual_seed(3)
    y = (torch.randn(T, batch, device="cuda", generator=g).cumsum(0) * 0.5).contiguous()
    y[:, torch.as_tensor(idx, device="cuda")] = dev(ys)
    out = ctx.hgf_filter(y, iters=iters)
    ref = hgf.hgf_filter(ys, iters=iters)
    got = out[:, :, torch.as_tensor(idx, device="cuda")].cpu().numpy()
    names = ("m_x", "v_x", "m_z", "v_z")
    rep = {n: (float(rel_l2(got[:, k], ref[:, k])), float(np.abs(got[:, k] - ref[:, k]).max())) for k, n in enumerate(names)}
    print("HGF configs[3] parity (relL2, max abs):", rep)
    assert rep["m_x"][0] < HGF_TOL["m_x"] and rep["v_x"][0] < HGF_TOL["v_x"]
    assert rep["m_z"][0] < HGF_TOL["m_z"] and rep["v_z"][0] < HGF_TOL["v_z"]


def test_vmp_gamma_precision_free_energy(ctx):
    """rxg_lgssm_vmp_gamma_fe_f32: Bethe free energy per iteration against the oracle's evaluation of the definition
    (dense q(x)); non-increasing over the iterations, as the reference asserts for its VMP models."""
    rng = np.random.default_rng(14)
    T, batch = 120, 33
    x = np.cumsum(rng.standard_normal((T, batch)), axis=0)
    y = (x + rng.standard_normal((T, batch)) / np.sqrt(rng.gamma(2.0, 1.0, batch) + 0.2)).astype(np.float32)
    ref = vmp.lgssm_gamma_precision(y, iterations=7, return_free_energy=True)
    r = ctx.lgssm_vmp_gamma(dev(y), iterations=7, want_free_energy=True)
    fe = r["free_energy"].cpu().numpy()
    assert fe.shape == (7, batch)
    err = np.abs(fe - ref["free_energy"]) / np.abs(ref["free_energy"])
    print("vmp gamma free energy rel err max", err.max())
    assert err.max() < 2e-5
    assert np.all(np.diff(fe, axis=0) < 1e-3 * np.abs(fe[:-1]))
    assert rel_l2(r["mean"].cpu().numpy(), ref["mean"]) < 1e-5


def test_vmp_gamma_precision(ctx):
    rng = np.random.default_rng(4)
    T, batch = 400, 70
    x = np.cumsum(rng.standard_normal((T, batch)), axis=0)
    tau = rng.gamma(2.0, 1.0, batch) + 0.2
    y = (x + rng.standard_normal((T, batch)) / np.sqrt(tau)).astype(np.float32)
    ref = vmp.lgssm_gamma_precision(y, iterations=8)
    r = ctx.lgssm_vmp_gamma(dev(y), iterations=8)
    assert rel_l2(r["mean"].cpu().numpy(), ref["mean"]) < 1e-5
    assert rel_l2(r["var"].cpu().numpy(), ref["var"]) < 1e-4
    assert rel_l2(r["rate"].cpu().numpy(), ref["rate"]) < 1e-4
    assert rel_l2(r["shape"].cpu().numpy(), ref["shape"]) < 1e-6


def test_stream_vmp_gamma_vs_oracle_and_chunks(rx, ctx):
    """Streaming mean-field VMP with a Gamma observation precision (the reference's test_model1): CUDA vs fp64 oracle,
    free energy included; time-chunks with the carry are bitwise the single call; engine mirror."""
    rng = np.random.default_rng(3)
    n, batch = 40, 200
    x = np.cumsum(rng.standard_normal((n, batch)), axis=0)
    y = (x + rng.standard_normal((n, batch)) / np.sqrt(10.0)).astype(np.float32)
    ref, rfe = vmp.stream_vmp_gamma(y.astype(np.float64), iterations=4, return_free_energy=True)
    out, fe = ctx.stream_vmp_gamma(dev(y), iters=4, want_free_energy=True)
    o = out.cpu().numpy()
    assert rel_l2(o[:, 0], ref[:, 0]) < 1e-5 and rel_l2(o[:, 1], ref[:, 1]) < 1e-5
    assert np.array_equal(o[:, 2], ref[:, 2].astype(np.float32)) and rel_l2(o[:, 3], ref[:, 3]) < 1e-5
    assert np.max(np.abs(fe.cpu().numpy() - rfe)) < 2e-3 * np.max(np.abs(rfe))
    hist = fe.double().mean(dim=0)                           # reference: averaged over observations, per iteration
    assert torch.all(hist[1:] - hist[:-1] <= 1e-4)           # inference_tests.jl:846 (fp32 slack)
    parts, prev = [], None
    for a, b in ((0, 1), (1, 17), (17, 40)):
        p, _ = ctx.stream_vmp_gamma(dev(y[a:b]), iters=4, prev=prev)
        prev = p[-1].contiguous()
        parts.append(p)
    assert torch.equal(torch.cat(parts), out)
    eng = rx.infer(model=rx.kalman_gamma_streaming(), datastream=[dev(y[:9]), dev(y[9:])], batch=batch, iterations=4,
                   keephistory=n, free_energy=True, context=ctx)
    assert torch.equal(eng.history["x_t"].mean(), out[:, 0]) and torch.equal(eng.history["τ"].rate(), out[:, 3])
    assert eng.free_energy_history.shape == (4, batch)
    res = rx.infer(model=rx.kalman_gamma_streaming(), data={"y": dev(y)}, iterations=4, free_energy=True, context=ctx)
    assert torch.equal(res.history["τ"].shape(), out[:, 2])
