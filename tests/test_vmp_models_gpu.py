"""The five small fused VMP kernels against their fp64 oracles, chain by chain, at non-default hyper-parameters:
hgf_filter_kernel and the three GCV rule kernels (oracle/hgf.py, oracle/rules.py), vmp_gamma_kernel
(vmp.lgssm_gamma_precision), stream_vmp_gamma_kernel (vmp.stream_vmp_gamma), ar_vmp_kernel<4|8> (vmp.ar_regression) and
mv_iid_wishart_vmp_kernel<1..6> (vmp.mv_iid_wishart).

Every chain gets its own data and the oracle sees the fp32-rounded inputs the device saw.  Each output is gated per chain
(``gate``), so one wrong chain fails the case and the message names it.  The hyper-parameter sets avoid 1 and 0, so that
kappa vs kappa^2, a vs a^2, w vs 1/w, a dropped omega, log w, p log w0 or xi0 term each move the outputs far beyond the
bounds.  A reversed batch must give the reversed outputs bit for bit (one thread per chain, one code path).  The refusals
of the C entries close the file."""
import ctypes

import numpy as np
import pytest
import torch
from scipy.signal import lfilter

from oracle import hgf, vmp
from oracle import rules as R

pytestmark = pytest.mark.gpu

WORST = {}                  # (kernel, output) -> worst per-chain error over the session, printed at the end (pytest -s)


@pytest.fixture(scope="module", autouse=True)
def _report_worst():
    yield
    for (kern, out), e in sorted(WORST.items()):
        print(f"worst per-chain error  {kern:16s} {out:12s} {e:.3g}")


def f32(a):
    return np.asarray(a, np.float32).astype(np.float64)


def fl(v):
    return float(np.float32(v))


def dev(a):
    return torch.as_tensor(np.ascontiguousarray(a), dtype=torch.float32, device="cuda")


def chain_err(got, ref, floor):
    """err_c = ||got[..., c] - ref[..., c]|| / max(||ref[..., c]||, floor sqrt(n)), chains on the last axis, n entries
    per chain: relative L2 per chain; ``floor`` is an RMS floor for outputs that can be near zero."""
    g = np.asarray(got, np.float64)
    r = np.asarray(ref, np.float64)
    assert g.shape == r.shape, (g.shape, r.shape)
    g = g.reshape(-1, g.shape[-1])
    r = r.reshape(-1, r.shape[-1])
    return np.linalg.norm(g - r, axis=0) / np.maximum(np.linalg.norm(r, axis=0), floor * np.sqrt(r.shape[0]))


def gate(kern, case, name, got, ref, tol, floor=1e-3):
    if isinstance(got, torch.Tensor):
        got = got.cpu().numpy()
    e = chain_err(got, ref, floor)
    c = int(np.argmax(np.where(np.isnan(e), np.inf, e)))
    WORST[(kern, name)] = max(WORST.get((kern, name), 0.0), float(e[c]))
    assert e[c] <= tol, f"{kern} {case}: {name} worst chain {c}: error {e[c]:.3g} > {tol:g}"


def flip(t):
    return torch.flip(t, [-1]).contiguous()


# ====================================================================================== HGF filter
# (kappa, omega, z_variance, y_variance, init = (m_z, v_z, m_x, v_x)); parameters are fp32-exact after fl()
HGF_SETS = {
    "default": (1.0, 0.0, 0.04, 0.01, (0.0, 5.0, 0.0, 5.0)),
    "k0.6,w-0.8": (0.6, -0.8, 0.0625, 0.015625, (0.3, 2.5, -0.4, 3.0)),
    "k1.7,w0.5": (1.7, 0.5, 0.015625, 0.03125, (-0.5, 1.5, 0.8, 4.0)),
}
# per chain, relative L2 over T (RMS floor 1e-3 for the means); the free energy relative to max(RMS, 1) over (T, iters).
# HGF_TOL of test_vmp_hgf_gpu.py, now per chain
HGF_TOL = {"m_x": 1e-6, "v_x": 2e-6, "m_z": 5e-6, "v_z": 5e-6, "fe": 2e-5}
HGF_OUT = ("m_x", "v_x", "m_z", "v_z")


def _hgf_params(name):
    k, w, zv, yv, init = HGF_SETS[name]
    return dict(kappa=fl(k), omega=fl(w), z_variance=fl(zv), y_variance=fl(yv)), tuple(fl(v) for v in init)


@pytest.mark.parametrize("T", [1, 37, 200])
@pytest.mark.parametrize("pset", list(HGF_SETS))
def test_hgf_filter_per_chain(ctx, pset, T):
    p, init = _hgf_params(pset)
    for batch in (1, 65, 130):                                      # tails of the 64-thread block
        _, _, y = hgf.generate_data(T, batch, seed=T + batch, **p)
        for iters in (1, 10):
            case = f"{pset} T={T} batch={batch} iters={iters}"
            out, fe = ctx.hgf_filter(dev(y), iters=iters, init=init, want_free_energy=True, **p)
            ref, fe_ref = hgf.hgf_filter(y, iters=iters, init=init, return_free_energy=True, **p)
            o = out.cpu().numpy()
            for k, n in enumerate(HGF_OUT):
                gate("hgf", case, n, o[:, k], ref[:, k], HGF_TOL[n])
            gate("hgf", case, "free_energy", fe, fe_ref, HGF_TOL["fe"], floor=1.0)
            assert torch.equal(ctx.hgf_filter(dev(y), iters=iters, init=init, **p), out), case   # FE does not perturb
            if batch == 130:
                ro, rf = ctx.hgf_filter(flip(dev(y)), iters=iters, init=init, want_free_energy=True, **p)
                assert torch.equal(flip(ro), out) and torch.equal(flip(rf), fe), case


@pytest.mark.parametrize("pset", list(HGF_SETS))
def test_hgf_chunks_with_prev(ctx, pset):
    """A stream cut into chunks, each continuing from prev = out[-1] of the last, is bitwise the single call."""
    p, init = _hgf_params(pset)
    _, _, y = hgf.generate_data(120, 97, seed=11, **p)
    out, fe = ctx.hgf_filter(dev(y), iters=6, init=init, want_free_energy=True, **p)
    o1, f1 = ctx.hgf_filter(dev(y[:37]), iters=6, init=init, want_free_energy=True, **p)
    o2, f2 = ctx.hgf_filter_chunk(dev(y[37:38]), o1[-1].contiguous(), iters=6, want_free_energy=True, **p)
    o3, f3 = ctx.hgf_filter_chunk(dev(y[38:]), o2[-1].contiguous(), iters=6, want_free_energy=True, **p)
    assert torch.equal(torch.cat([o1, o2, o3]), out) and torch.equal(torch.cat([f1, f2, f3]), fe)


# ====================================================================================== GCV rule kernels
GCV_TOL = {"out_v": 1e-6, "yx_m": 1e-6, "yx_V": 1e-6, "z_m": 2e-5, "z_v": 5e-5}


@pytest.mark.parametrize("pset", list(HGF_SETS))
def test_gcv_rules_per_message(ctx, pset):
    p, _ = _hgf_params(pset)
    k, w = p["kappa"], p["omega"]
    rng = np.random.default_rng(len(pset))
    n = 2050                                                        # ragged against the 256- and 128-thread blocks
    my, vy = f32(rng.standard_normal(n)), f32(rng.random(n) * 0.1 + 0.01)
    mx, vx = f32(rng.standard_normal(n)), f32(rng.random(n) + 0.1)
    mz, vz = f32(rng.standard_normal(n) * 0.5), f32(rng.random(n) * 0.5 + 0.05)
    mo, vo = ctx.rule_gcv_out(dev(mx), dev(vx), dev(mz), dev(vz), k, w)
    rmo, rvo = R.gcv_y((mx, vx), (mz, vz), k, w)
    assert np.array_equal(mo.cpu().numpy(), mx.astype(np.float32)), pset
    gate("gcv_out", pset, "v", vo.cpu().numpy()[None], rvo[None], GCV_TOL["out_v"])
    m, V = ctx.marginalrule_gcv_yx(dev(my), dev(vy), dev(mx), dev(vx), dev(mz), dev(vz), k, w)
    rm, rV = R.gcv_marginal_yx((my, vy), (mx, vx), (mz, vz), k, w)
    gate("gcv_yx", pset, "m", m, rm.T, GCV_TOL["yx_m"])
    gate("gcv_yx", pset, "V", V, np.moveaxis(rV, 0, -1), GCV_TOL["yx_V"])
    # the z product from the fp32-rounded exact joint, so that only this kernel is measured
    jm, jV = f32(rm.T), f32(np.moveaxis(rV, 0, -1))
    zp_m, zp_v = f32(rng.standard_normal(n) * 0.3), f32(rng.random(n) * 0.5 + 0.05)
    gz, gv = ctx.rule_gcv_z_prod(dev(jm), dev(jV), dev(zp_m), dev(zp_v), k, w)
    rz, rv = R.prod_normal_elq((zp_m, zp_v), R.gcv_z_elq(jm.T, np.moveaxis(jV, -1, 0), k, w))
    gate("gcv_z_prod", pset, "m_z", gz.cpu().numpy()[None], rz[None], GCV_TOL["z_m"], floor=0.1)
    gate("gcv_z_prod", pset, "v_z", gv.cpu().numpy()[None], rv[None], GCV_TOL["z_v"])
    # message order reversed -> outputs reversed, bit for bit
    rev = lambda a: dev(a[..., ::-1])
    assert torch.equal(flip(ctx.rule_gcv_out(rev(mx), rev(vx), rev(mz), rev(vz), k, w)[1]), vo)
    m2, V2 = ctx.marginalrule_gcv_yx(rev(my), rev(vy), rev(mx), rev(vx), rev(mz), rev(vz), k, w)
    assert torch.equal(flip(m2), m) and torch.equal(flip(V2), V)
    z2, v2 = ctx.rule_gcv_z_prod(rev(jm), rev(jV), rev(zp_m), rev(zp_v), k, w)
    assert torch.equal(flip(z2), gz) and torch.equal(flip(v2), gv)


# ====================================================================================== Gamma VMP around the smoother
GAMMA_SETS = {
    "default": dict(a=1.0, v_proc=1.0, prior=(0.0, 100.0), gamma_prior=(1.0, 1.0), init_E_tau=1.0),
    "a-0.9": dict(a=-0.9, v_proc=0.6, prior=(1.5, 2.0), gamma_prior=(2.0, 3.0), init_E_tau=0.4),
    "a0.7": dict(a=0.7, v_proc=1.8, prior=(1.5, 2.0), gamma_prior=(2.0, 3.0), init_E_tau=0.4),
}
# test_vmp_hgf_gpu.py's bounds, per chain: mean 1e-5, var / rate 1e-4, shape 1e-6, free energy 2e-5 (relative to max(|F|, 1))
GAMMA_TOL = {"mean": 1e-5, "var": 1e-4, "shape": 1e-6, "rate": 1e-4, "free_energy": 2e-5}


def _gamma_data(T, batch, a, v_proc, seed):
    rng = np.random.default_rng(seed)
    x = np.zeros((T, batch))
    x[0] = 1.5 + np.sqrt(2.0) * rng.standard_normal(batch)
    for t in range(1, T):
        x[t] = a * x[t - 1] + np.sqrt(v_proc) * rng.standard_normal(batch)
    tau = rng.gamma(2.0, 1.0, batch) + 0.2                          # every chain its own observation precision
    return f32(x + rng.standard_normal((T, batch)) / np.sqrt(tau))


@pytest.mark.parametrize("T", [1, 2, 150])
@pytest.mark.parametrize("pset", list(GAMMA_SETS))
def test_lgssm_vmp_gamma_per_chain(ctx, pset, T):
    s = GAMMA_SETS[pset]
    a, vp, pr, gp, e0 = fl(s["a"]), fl(s["v_proc"]), tuple(map(fl, s["prior"])), tuple(map(fl, s["gamma_prior"])), fl(s["init_E_tau"])
    batch = 130                                                     # tail of the 128-thread block
    y = _gamma_data(T, batch, a, vp, seed=T)
    for its in (1, 8):
        case = f"{pset} T={T} iterations={its}"
        kw = dict(iterations=its, a=a, v_proc=vp, prior=pr, gamma_prior=gp, init_E_tau=e0)
        r = ctx.lgssm_vmp_gamma(dev(y), want_free_energy=True, **kw)
        ref = vmp.lgssm_gamma_precision(y, A_scalar=a, prior=pr, proc_var=vp, gamma_prior=gp, iterations=its,
                                        init_Etau=e0, return_free_energy=True)
        for k in ("mean", "var"):
            gate("lgssm_vmp_gamma", case, k, r[k], ref[k], GAMMA_TOL[k])
        for k in ("shape", "rate"):
            gate("lgssm_vmp_gamma", case, k, r[k].cpu().numpy()[None], np.broadcast_to(ref[k], (batch,))[None], GAMMA_TOL[k])
        gate("lgssm_vmp_gamma", case, "free_energy", r["free_energy"], ref["free_energy"], GAMMA_TOL["free_energy"], floor=1.0)
        plain = ctx.lgssm_vmp_gamma(dev(y), **kw)
        for k in ("mean", "var", "shape", "rate"):
            assert torch.equal(plain[k], r[k]), (case, k)             # the free energy does not perturb the posteriors
        rr = ctx.lgssm_vmp_gamma(flip(dev(y)), want_free_energy=True, **kw)
        for k in ("mean", "var", "shape", "rate", "free_energy"):
            assert torch.equal(flip(rr[k]), r[k]), (case, k)


# ====================================================================================== streaming Gamma model
STREAM_SETS = {"default": (1.0, (0.0, 1e3, 1.0, 1.0)), "w0.3": (0.3, (0.5, 20.0, 2.0, 1.5)), "w3": (3.0, (-0.7, 4.0, 3.5, 0.6))}
# test_vmp_hgf_gpu.py's 1e-5 for m_x, v_x, rate, per chain; shape is exact (a_p + 1/2 per datum)
STREAM_TOL = {"m_x": 1e-5, "v_x": 1e-5, "rate": 1e-5, "free_energy": 2e-5}


@pytest.mark.parametrize("pset", list(STREAM_SETS))
def test_stream_vmp_gamma_per_chain_and_chunks(ctx, pset):
    w, init = STREAM_SETS[pset]
    w, init = fl(w), tuple(fl(v) for v in init)
    rng = np.random.default_rng(int(w * 10))
    T, batch = 60, 200
    x = np.cumsum(rng.standard_normal((T, batch)) / np.sqrt(w), axis=0)
    y = f32(x + rng.standard_normal((T, batch)) / np.sqrt(rng.gamma(2.0, 1.0, batch) + 0.2))
    for its in (1, 4):
        case = f"{pset} iterations={its}"
        out, fe = ctx.stream_vmp_gamma(dev(y), iters=its, w=w, init=init, want_free_energy=True)
        ref, rfe = vmp.stream_vmp_gamma(y, iterations=its, w=w, init_x=init[:2], init_tau=init[2:], return_free_energy=True)
        o = out.cpu().numpy()
        gate("stream_vmp_gamma", case, "m_x", o[:, 0], ref[:, 0], STREAM_TOL["m_x"])
        gate("stream_vmp_gamma", case, "v_x", o[:, 1], ref[:, 1], STREAM_TOL["v_x"])
        assert np.array_equal(o[:, 2], ref[:, 2].astype(np.float32)), case
        gate("stream_vmp_gamma", case, "rate", o[:, 3], ref[:, 3], STREAM_TOL["rate"])
        gate("stream_vmp_gamma", case, "free_energy", fe, rfe, STREAM_TOL["free_energy"], floor=1.0)
        ro, rf = ctx.stream_vmp_gamma(flip(dev(y)), iters=its, w=w, init=init, want_free_energy=True)
        assert torch.equal(flip(ro), out) and torch.equal(flip(rf), fe), case
        parts, fparts, prev = [], [], None
        for lo, hi in ((0, 1), (1, 17), (17, T)):
            p, f = ctx.stream_vmp_gamma(dev(y[lo:hi]), iters=its, w=w, init=init, prev=prev, want_free_energy=True)
            prev = p[-1].contiguous()
            parts.append(p); fparts.append(f)
        assert torch.equal(torch.cat(parts), out) and torch.equal(torch.cat(fparts), fe), case


# ====================================================================================== AR regression VMP
# (gamma_prior, theta_prior_precision, init_gamma)
AR_SETS = {"default": ((1.0, 1.0), 1.0, (1.0, 1.0)), "set1": ((2.5, 0.5), 0.3, (3.0, 2.0)), "set2": ((0.7, 4.0), 5.0, (0.5, 2.5))}
# fp64 in the kernel, fp32 outputs: per chain 1e-6 on the fp32 outputs; 1e-9 relative on the fp64 free energy (tighter
# than the 1e-7 of test_reference_rng_goldens.py; worst chain measured on an H100 80GB HBM3: 8.7e-11)
AR_TOL = {"theta_mean": 1e-6, "theta_cov": 1e-6, "gamma_shape": 1e-6, "gamma_rate": 1e-6, "free_energy": 1e-9}


def _ar_series(N, batch, order, seed):
    """Distinct series per chain: white noise with its own scale and offset (every 3rd chain), and AR(q) series,
    1 <= q <= order, with their own stable coefficients (roots drawn inside the unit circle) and innovation scale."""
    rng = np.random.default_rng(seed)
    s = np.zeros((N, batch))
    for c in range(batch):
        scale = 0.3 + 2.0 * rng.random()
        if c % 3 == 0:
            s[:, c] = rng.normal(0.5 * rng.standard_normal(), scale, N)
            continue
        q = 1 + rng.integers(order)
        ar = np.poly(rng.uniform(-0.85, 0.85, q))                 # x_k = -sum_j ar[j] x_{k-j} + e_k
        s[:, c] = lfilter([1.0], ar, scale * rng.standard_normal(N + 50))[50:]
    return f32(s)


@pytest.mark.parametrize("order", range(1, 9))
def test_ar_vmp_per_chain(ctx, order):
    for N in (order + 1, order + 7, 1000):
        for batch in (1, 127, 129):
            s = _ar_series(N, batch, order, seed=1000 * order + N + batch)
            for pset, (gp, w0, ig) in AR_SETS.items():
                gp, w0, ig = tuple(map(fl, gp)), fl(w0), tuple(map(fl, ig))
                for its in (1, 15):
                    case = f"{pset} order={order} N={N} batch={batch} iterations={its}"
                    kw = dict(iterations=its, gamma_prior=gp, theta_prior_precision=w0, init_gamma=ig)
                    r = ctx.ar_vmp(dev(s), order, **kw)
                    ref = vmp.ar_regression(s, order, **kw)
                    gate("ar_vmp", case, "theta_mean", r["theta_mean"], ref["theta_mean"], AR_TOL["theta_mean"])
                    gate("ar_vmp", case, "theta_cov", r["theta_cov"], ref["theta_cov"], AR_TOL["theta_cov"])
                    for k in ("gamma_shape", "gamma_rate"):
                        gate("ar_vmp", case, k, r[k].cpu().numpy()[None], ref[k][None], AR_TOL[k])
                    gate("ar_vmp", case, "free_energy", r["free_energy"], ref["free_energy"], AR_TOL["free_energy"], floor=1.0)
                    if batch == 129 and its == 15:
                        nf = ctx.ar_vmp(dev(s), order, want_free_energy=False, **kw)
                        rr = ctx.ar_vmp(flip(dev(s)), order, **kw)
                        for k in ("theta_mean", "theta_cov", "gamma_shape", "gamma_rate"):
                            assert torch.equal(nf[k], r[k]), (case, k)
                        for k in ("theta_mean", "theta_cov", "gamma_shape", "gamma_rate", "free_energy"):
                            assert torch.equal(flip(rr[k]), r[k]), (case, k)


# ====================================================================================== IID Wishart VMP
def _spd(rng, d, scale, jitter):
    M = rng.standard_normal((d, d))
    return scale * (M @ M.T / d + jitter * np.eye(d))


def _iid_priors(d, pset):
    """(mu0, Lambda0, nu0, inv_scale0, init_E_P), fp32-exact.  The default set is the reference test's, with the mean of
    vague(Wishart, d) as the initial E[P]."""
    if pset == "default":
        return f32(np.zeros(d)), f32(100.0 * np.eye(d)), d + 1.0, f32(np.eye(d)), f32(d * 1e12 * np.eye(d))
    rng = np.random.default_rng(7 * d + len(pset))
    if pset == "set1":
        return (f32(np.linspace(-0.7, 1.3, d)), f32(_spd(rng, d, 2.5, 0.5)), d + 2.5, f32(_spd(rng, d, 0.6, 0.3)),
                f32(np.linalg.inv(_spd(rng, d, 0.8, 0.4))))
    return (f32(np.linspace(1.1, -0.4, d) + 0.3), f32(_spd(rng, d, 0.4, 0.2)), d - 0.5, f32(_spd(rng, d, 3.0, 0.5)),
            f32(_spd(rng, d, 1.5, 0.5)))


# fp64 in the kernel, fp32 outputs: per chain 1e-6 (relative L2 / Frobenius); df exact
IID_TOL = {"m_mean": 1e-6, "m_cov": 1e-6, "inv_scale": 1e-6}


@pytest.mark.parametrize("d", range(1, 7))
def test_mv_iid_wishart_vmp_per_chain(ctx, d):
    batch = 130
    for pset in ("default", "set1", "set2"):
        mu0, L0, nu0, iS0, EP0 = _iid_priors(d, pset)
        for N in (1, 2, 300):
            rng = np.random.default_rng(100 * d + N)
            ys = []
            for _ in range(batch):                                   # every data set its own mean and covariance
                C = _spd(rng, d, 0.5 + rng.random(), 0.1)
                ys.append(rng.standard_normal(d)[None, :] + rng.standard_normal((N, d)) @ np.linalg.cholesky(C).T)
            y = f32(np.stack(ys, axis=-1))
            for its in (1, 8):
                case = f"{pset} d={d} N={N} iterations={its}"
                kw = dict(iterations=its, mu0=mu0, Lambda0=L0, nu0=nu0, inv_scale0=iS0, init_E_P=EP0)
                r = ctx.mv_iid_wishart_vmp(dev(y), **kw)
                ref = vmp.mv_iid_wishart(y, **kw)
                assert int(r["status"].abs().sum()) == 0, (case, r["status"].nonzero())
                for k in ("m_mean", "m_cov", "inv_scale"):
                    gate("mv_iid_wishart", case, k, r[k], ref[k], IID_TOL[k])
                assert np.array_equal(r["df"].cpu().numpy(), ref["df"].astype(np.float32)), case
                if N == 300 and its == 8:
                    rr = ctx.mv_iid_wishart_vmp(flip(dev(y)), **kw)
                    for k in ("m_mean", "m_cov", "df", "inv_scale", "status"):
                        assert torch.equal(flip(rr[k]), r[k]), (case, k)


# ====================================================================================== refusals
def _code(fn, *a, **k):
    from rxinfer_jl_b200 import _lib as L
    with pytest.raises(L.RxGaussError) as e:
        fn(*a, **k)
    return e.value.code


def test_refusals(ctx):
    from rxinfer_jl_b200 import _lib as L
    U, BAD = L.RXG_ERR_UNSUPPORTED, L.RXG_ERR_BAD_ARG
    y = dev(np.zeros((12, 3)))
    # ar_vmp: orders 1..8, N > order, iterations >= 1, positive priors
    assert _code(ctx.ar_vmp, y, 0) == U and _code(ctx.ar_vmp, y, 9) == U
    assert _code(ctx.ar_vmp, y[:5].contiguous(), 5) == BAD
    ctx.ar_vmp(y[:6].contiguous(), 5)                               # N = order + 1: one regression row
    assert _code(ctx.ar_vmp, y, 2, iterations=0) == BAD
    for kw in (dict(gamma_prior=(0.0, 1.0)), dict(gamma_prior=(1.0, -1.0)), dict(theta_prior_precision=0.0),
               dict(init_gamma=(-1.0, 1.0)), dict(init_gamma=(1.0, float("nan")))):
        assert _code(ctx.ar_vmp, y, 2, **kw) == BAD, kw
    # mv_iid_wishart_vmp: d in 1..6, N and iterations >= 1, nu0 > d - 1
    assert _code(ctx.mv_iid_wishart_vmp, dev(np.zeros((4, 7, 3)))) == U
    assert _code(ctx.mv_iid_wishart_vmp, dev(np.zeros((4, 0, 3)))) == BAD
    assert _code(ctx.mv_iid_wishart_vmp, dev(np.zeros((0, 2, 3)))) == BAD
    assert _code(ctx.mv_iid_wishart_vmp, dev(np.ones((4, 2, 3))), iterations=0) == BAD
    for nu0 in (1.0, 0.5, -3.0, float("nan")):
        assert _code(ctx.mv_iid_wishart_vmp, dev(np.ones((4, 2, 3))), nu0=nu0) == BAD, nu0
    assert int(ctx.mv_iid_wishart_vmp(dev(np.ones((4, 2, 3))), nu0=1.25)["status"].abs().sum()) == 0
    # lgssm_vmp_gamma: T, iterations >= 1; v_proc, v0, a0, b0, init_E_tau > 0
    assert _code(ctx.lgssm_vmp_gamma, y, iterations=0) == BAD
    assert _code(ctx.lgssm_vmp_gamma, dev(np.zeros((0, 3)))) == BAD
    for kw in (dict(v_proc=0.0), dict(v_proc=-1.0), dict(prior=(0.0, 0.0)), dict(prior=(0.0, -2.0)),
               dict(gamma_prior=(0.0, 1.0)), dict(gamma_prior=(-1.0, 1.0)), dict(gamma_prior=(1.0, 0.0)),
               dict(gamma_prior=(1.0, -1.0)), dict(init_E_tau=0.0), dict(init_E_tau=-0.5), dict(v_proc=float("nan"))):
        assert _code(ctx.lgssm_vmp_gamma, y, want_free_energy=True, **kw) == BAD, kw
    # stream_vmp_gamma: iterations >= 1, w > 0
    for kw in (dict(iters=0), dict(w=0.0), dict(w=-1.0)):
        assert _code(ctx.stream_vmp_gamma, y, **kw) == BAD, kw
    # hgf_filter: iterations >= 1, positive variances
    for kw in (dict(iters=0), dict(z_variance=0.0), dict(y_variance=-0.01)):
        assert _code(ctx.hgf_filter, y, **kw) == BAD, kw
    # host pointers
    h = torch.zeros(4096)
    hp = lambda: L.as_fp(h.data_ptr())
    dp = ctypes.cast(ctypes.c_void_p(h.data_ptr()), ctypes.POINTER(ctypes.c_double))
    ini = (ctypes.c_float * 4)(0.0, 1.0, 1.0, 1.0)
    eye = np.eye(2, dtype=np.float32).ravel()
    z2 = np.zeros(2, np.float32)
    e = lambda a: a.ctypes.data_as(L.fp)
    i32 = ctypes.cast(ctypes.c_void_p(h.data_ptr()), L.i32p)
    assert ctx.lib.rxg_ar_vmp_f32(ctx.h, 2, 12, 3, 2, 1.0, 1.0, 1.0, 1.0, 1.0, hp(), hp(), hp(), hp(), hp(), dp, 0) == U
    assert ctx.lib.rxg_mv_iid_wishart_vmp_f32(ctx.h, 2, 4, 3, 2, e(z2), e(eye), 3.0, e(eye), e(eye), hp(), hp(), hp(), hp(),
                                              hp(), i32, 0) == U
    assert ctx.lib.rxg_lgssm_vmp_gamma_fe_f32(ctx.h, 12, 3, 2, 1.0, 1.0, 0.0, 100.0, 1.0, 1.0, 1.0, hp(), hp(), hp(), hp(),
                                              hp(), hp(), 0) == U
    assert ctx.lib.rxg_stream_vmp_gamma_f32(ctx.h, 12, 3, 2, 1.0, ctypes.cast(ini, L.fp), L.as_fp(0), hp(), hp(), hp(), 0) == U
    assert ctx.lib.rxg_hgf_filter_fe_f32(ctx.h, 12, 3, 2, 1.0, 0.0, 0.04, 0.01, ctypes.cast(ini, L.fp), L.as_fp(0), hp(), hp(),
                                         hp(), 0) == U
    assert ctx.lib.rxg_rule_gcv_out_f32(ctx.h, 8, hp(), hp(), hp(), hp(), 1.0, 0.0, hp(), hp(), 0) == U
    assert ctx.lib.rxg_marginalrule_gcv_yx_f32(ctx.h, 8, hp(), hp(), hp(), hp(), hp(), hp(), 1.0, 0.0, hp(), hp(), 0) == U
    assert ctx.lib.rxg_rule_gcv_z_prod_f32(ctx.h, 8, hp(), hp(), hp(), hp(), 1.0, 0.0, hp(), hp(), 0) == U
    assert ctx.lib.rxg_rule_gcv_out_f32(ctx.h, -1, hp(), hp(), hp(), hp(), 1.0, 0.0, hp(), hp(), L.PTR_DEVICE) == BAD
