"""Bayesian multinomial regression (MultinomialPolya, mean-field Pólya-Gamma VMP; DESIGN 3.22), CPU only: the fp64
reference of oracle/multinomial.py against the stick-breaking identity, the binomial reference at K = 2, the uncollapsed
bound and quadrature evidence; its free energy never increases offline; the collapsed Sherman–Morrison step against the
dense one; the reference test's assertions (multinomialreg_tests.jl) on the reference; the kernel bodies compiled for the
host (tests/c/multinomial_host_harness.cu) against the reference at K = 2 … 64, chunked online runs against one run; and
the argument handling of ``infer``."""
import ctypes
import os
import shutil
import subprocess

import numpy as np
import pytest
from scipy.special import gammaln, softmax
from scipy.stats import binom, multinomial, wishart

from oracle import binomial as ob
from oracle import multinomial as om
from util import TOL_COV, TOL_MEAN

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FE_TOL = 1e-5


def random_problem(K, n, nb, seed, max_trials=20, zero_rows=0.1):
    """Counts y [n, K, nb] int32 (about zero_rows of the samples all-zero) and a prior xi0 [D], W0 [D, D]."""
    rng = np.random.default_rng(seed)
    D = K - 1
    y = np.zeros((n, K, nb), np.int32)
    for b in range(nb):
        p = softmax(rng.standard_normal(K))
        N = rng.integers(0, max_trials + 1, n) * (rng.random(n) >= zero_rows)
        y[:, :, b] = np.array([rng.multinomial(t, p) for t in N])
    A = rng.standard_normal((D, D))
    return y, 0.3 * rng.standard_normal(D), A @ A.T / D + np.eye(D)


def f32(a):
    return np.asarray(a, np.float32).astype(np.float64)


def reference_on_f32(y, xi0, W0, its):
    """The fp64 reference of every chain on the inputs the kernel sees (the prior rounded to fp32)."""
    return om.vmp_batch(y, f32(xi0), f32(W0), its)


def online_reference_on_f32(y, xi0, W0, its=1):
    return om.online_batch(y, f32(xi0), f32(W0), its)


def gate(case, r, ref, chains=None, fe=True):
    """Per chain: mean at TOL_MEAN and covariance at TOL_COV relative L2 over the iterations (or data), F at FE_TOL
    relative to max(|F|, 1).  Returns the worst errors."""
    nb = ref["hist_mean"].shape[-1]
    worst = {}
    for b in range(nb) if chains is None else chains:
        for key, tol in (("hist_mean", TOL_MEAN), ("hist_cov", TOL_COV)):
            if r.get(key) is None:
                continue
            a, e = np.asarray(r[key], np.float64)[..., b], ref[key][..., b]
            err = np.linalg.norm(a - e) / max(np.linalg.norm(e), 1e-30)
            assert err < tol, f"{case}: chain {b} {key} {err:.3g}"
            worst[key] = max(worst.get(key, 0.0), err)
        if fe:
            a, e = np.asarray(r["free_energy"])[:, b], ref["free_energy"][:, b]
            err = (np.abs(a - e) / np.maximum(np.abs(e), 1.0)).max()
            assert err < FE_TOL, f"{case}: chain {b} free energy {err:.3g}"
            worst["free_energy"] = max(worst.get("free_energy", 0.0), err)
    return worst


# ---------------------------------------------------------------- the reference against first principles
def test_stick_breaking_binomials_are_the_multinomial():
    rng = np.random.default_rng(0)
    for K in (2, 3, 7, 40):
        psi = rng.standard_normal(K - 1)
        p = om.stick_breaking(psi)
        np.testing.assert_allclose(p.sum(), 1.0, rtol=1e-15)
        sig = 1 / (1 + np.exp(-psi))
        for _ in range(5):
            y = rng.multinomial(rng.integers(1, 30), softmax(rng.standard_normal(K)))[None]
            Nk, yk = om.binomials(y)
            lp = binom.logpmf(yk[0], Nk[0], sig).sum()
            np.testing.assert_allclose(lp, multinomial.logpmf(y[0], y.sum(), p), rtol=1e-12)
            np.testing.assert_allclose(om.log_coefficient(y)[0],
                                       (gammaln(Nk + 1) - gammaln(yk + 1) - gammaln(Nk - yk + 1)).sum(), rtol=1e-13)


def test_k_equal_two_is_the_binomial_regression_with_x_equal_one():
    y, xi0, W0 = random_problem(2, 60, 1, seed=1)
    y = y[..., 0]
    a = om.vmp(y, xi0, W0, 12)
    b = ob.vmp(np.ones((60, 1)), y[:, 0], y.sum(1), xi0, W0, 12)
    for k in ("mean", "cov", "free_energy"):
        np.testing.assert_allclose(a[k], b[k], rtol=1e-12, atol=1e-12)


def test_the_uncollapsed_bound_is_above_the_collapsed_one_with_equality_at_c():
    y, xi0, W0 = random_problem(5, 40, 1, seed=2)
    y = y[..., 0]
    r = om.vmp(y, xi0, W0, 3)
    m, S = r["mean"][-1], r["cov"][-1]
    S0 = np.linalg.inv(W0)
    m0 = S0 @ xi0
    c = np.sqrt(m ** 2 + np.diag(S))
    F = om.free_energy(y, m0, S0, m, S)
    np.testing.assert_allclose(om.free_energy_uncollapsed(y, m0, S0, m, S, c), F, rtol=1e-12)
    rng = np.random.default_rng(3)
    for _ in range(20):
        cq = c * np.exp(rng.normal(0, 0.7, c.shape)) + rng.uniform(0, 0.1, c.shape)
        assert om.free_energy_uncollapsed(y, m0, S0, m, S, cq) >= F - 1e-12


def _log_evidence_quadrature(y, xi0, W0):
    """log p(y) on a grid, K = 2 or 3 (D = 1 or 2)."""
    D = len(xi0)
    S0 = np.linalg.inv(W0)
    m0 = S0 @ xi0
    g = np.linspace(-8, 8, 2001 if D == 1 else 501)
    P = np.stack(np.meshgrid(*([g] * D), indexing="ij"), -1).reshape(-1, D) + m0
    d = P - m0
    lp = -0.5 * np.einsum("ij,jk,ik->i", d, W0, d) - 0.5 * D * np.log(2 * np.pi) + 0.5 * np.linalg.slogdet(W0)[1]
    Nk, yk = om.binomials(y)
    ll = (gammaln(Nk + 1) - gammaln(yk + 1) - gammaln(Nk - yk + 1)).sum() + \
        (yk.sum(0)[None] * P - Nk.sum(0)[None] * np.logaddexp(0, P)).sum(1)
    t = lp + ll
    return np.log(np.exp(t - t.max()).sum() * (g[1] - g[0]) ** D) + t.max()


@pytest.mark.parametrize("K", [2, 3])
def test_the_free_energy_bounds_minus_the_log_evidence(K):
    for seed in range(4):
        y, xi0, W0 = random_problem(K, 6, 1, seed=10 + seed, max_trials=8, zero_rows=0.0)
        y = y[..., 0]
        r = om.vmp(y, xi0, W0, 30)
        assert r["free_energy"].min() >= -_log_evidence_quadrature(y, xi0, W0) - 1e-9


def test_the_free_energy_never_increases_offline():
    for K, seed in ((2, 0), (3, 1), (10, 2), (33, 3)):
        y, xi0, W0 = random_problem(K, 300, 3, seed=seed)
        fe = reference_on_f32(y, xi0, W0, 40)["free_energy"]
        assert (np.diff(fe, axis=0) <= 1e-9 * np.maximum(np.abs(fe[1:]), 1)).all()


def test_the_collapsed_sherman_morrison_step_is_the_dense_one():
    for K, seed in ((2, 4), (5, 5), (17, 6), (64, 7)):
        y, xi0, W0 = random_problem(K, 30, 1, seed=seed)
        y = y[..., 0].astype(np.float64)
        if K > 2:
            y[:, -2:] = 0                                         # the last category has no trials: d_D = 0 is skipped
        rng = np.random.default_rng(seed)
        S0 = np.linalg.inv(W0)
        m0 = S0 @ xi0
        A = rng.standard_normal((K - 1, K - 1))
        m, S = m0 + rng.standard_normal(K - 1), A @ A.T / K + 0.5 * np.eye(K - 1)     # any current q
        md, Sd = om.step(y, m0, S0, m, S)
        Nk, yk = om.binomials(y)
        mc, Sc, kl = om.collapsed_step((yk - Nk / 2).sum(0), Nk.sum(0), m0, S0, m, S)
        np.testing.assert_allclose(mc, md, rtol=1e-10, atol=1e-12)
        np.testing.assert_allclose(Sc, Sd, rtol=1e-10, atol=1e-13)
        np.testing.assert_allclose(kl, ob.kl_gauss(md, Sd, xi0, W0), rtol=1e-9, atol=1e-10)


def test_padding_with_all_zero_samples_drops_nothing():
    y, xi0, W0 = random_problem(6, 50, 2, seed=8)
    pad = np.concatenate([y, np.zeros((7, 6, 2), np.int32)])
    a, b = reference_on_f32(y, xi0, W0, 10), reference_on_f32(pad, xi0, W0, 10)
    for k in ("hist_mean", "hist_cov", "free_energy"):
        np.testing.assert_allclose(a[k], b[k], rtol=1e-12, atol=1e-12)


# ---------------------------------------------------------------- the reference test (multinomialreg_tests.jl)
def reference_offline(seed, K=10, N=20, nsamples=1000):
    """One data set of the offline item from a seeded numpy generator: ψ ~ N(0, I_K), p = softmax(ψ), nsamples draws of
    Multinomial(N, p), W_ψ ~ Wishart(K, I_{K-1}) (the reference's StableRNG samplers are not restated).  y [n, K]."""
    rng = np.random.default_rng(seed)
    p = softmax(rng.standard_normal(K))
    y = rng.multinomial(N, p, size=nsamples).astype(np.int32)
    W = wishart(df=K, scale=np.eye(K - 1)).rvs(random_state=rng)
    return y, W, p


def reference_online(seed=321, K=40, N=50, nsamples=5000):
    return reference_offline(seed, K, N, nsamples)


OFFLINE_SEEDS = range(20)


def offline_assertions(mean, fes, p, slack=1e-14):
    """The offline item's assertions on one data set: F[end] < F[1] and F[end] <= F[end-1] are asserted; returns whether
    mse(stick_breaking(mean ψ), p) < 2e-5 and |F[end-1] - F[end]| < 1e-8 hold.  Once converged, F[end] and F[end-1]
    differ by round-off of an F near 1e4, so the second comparison allows slack |F|: a few 1e-12 either way on the fp64
    reference; on the device the Sherman–Morrison step's round-off reaches F at up to 1e-11 relative (DESIGN 3.22)."""
    assert fes[-1] < fes[0] and fes[-1] <= fes[-2] + slack * abs(fes[-2])
    return np.mean((om.stick_breaking(mean) - p) ** 2) < 2e-5, abs(fes[-2] - fes[-1]) < 1e-8


# Of the 20 seeded data sets, the fp64 reference meets mse < 2e-5 on 15 and |dF| < 1e-8 on 15 (DESIGN 3.22: the W_ψ drawn
# from Wishart(K, I) shrinks the later sticks, and on some draws 100 iterations do not reach 1e-8).  Pinned here so that a
# change of the reference's fixed point or convergence shows.
OFFLINE_MSE_PASS, OFFLINE_CONVERGED = 15, 15


def test_the_offline_reference_assertions_on_the_fp64_reference():
    mse_pass = converged = 0
    for seed in OFFLINE_SEEDS:
        y, W, p = reference_offline(seed)
        r = om.vmp(y, np.zeros(9), W, 100)
        ok_mse, ok_conv = offline_assertions(r["mean"][-1], r["free_energy"], p)
        mse_pass += ok_mse
        converged += ok_conv
    assert (mse_pass, converged) == (OFFLINE_MSE_PASS, OFFLINE_CONVERGED)


def test_the_online_reference_assertions_on_the_fp64_reference():
    y, W, p = reference_online()
    r = om.online(y, np.zeros(39), W, 1)
    assert np.mean((om.stick_breaking(r["mean"][-1]) - p) ** 2) < 1e-3
    assert r["free_energy"][-1] < r["free_energy"][0]


# ---------------------------------------------------------------- the kernel bodies on the host
def _host_harness():
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    so = os.path.join(ROOT, "tests", "c", "_multinomial_host.so")
    src = os.path.join(ROOT, "tests", "c", "multinomial_host_harness.cu")
    hdrs = [os.path.join(ROOT, "rxinfer.jl_b200", "csrc", "rxg_multinomial.cuh")]
    if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(f) for f in [src] + hdrs):
        subprocess.run([nvcc, "-O2", "-Wno-deprecated-gpu-targets", "-shared", "-Xcompiler", "-fPIC", "-o", so, src], check=True)
    return ctypes.CDLL(so)


def _prior_block(xi0, W0):
    S0 = np.linalg.inv(f32(W0))
    return np.ascontiguousarray(np.concatenate([S0 @ f32(xi0), S0.ravel()]))


_P = lambda a: None if a is None else a.ctypes.data_as(ctypes.c_void_p)


def run_host(lib, y, xi0, W0, its):
    n, K, nb = y.shape
    D = K - 1
    z = lambda *s: np.zeros(s, np.float32)
    out = dict(psi_mean=z(D, nb), psi_cov=z(D, D, nb), free_energy=np.zeros((its, nb)), hist_mean=z(its, D, nb),
               hist_cov=z(its, D, D, nb), status=np.zeros(nb, np.int32))
    rc = lib.multinomial_host_vmp(K, n, ctypes.c_longlong(nb), its, _P(_prior_block(xi0, W0)),
                                  _P(np.ascontiguousarray(y, np.int32)),
                                  *(_P(out[k]) for k in ("psi_mean", "psi_cov", "free_energy", "hist_mean", "hist_cov",
                                                         "status")))
    assert rc == 0
    return out


def run_host_online(lib, y, xi0, W0, its=1, carry=None):
    """One call over y [T, K, nb]; carry = (m, S) fp64 is updated in place (None: start at the prior)."""
    T, K, nb = y.shape
    D = K - 1
    start = carry is None
    if start:
        carry = (np.zeros((D, nb)), np.zeros((D, D, nb)))
    out = dict(hist_mean=np.zeros((T, D, nb), np.float32), hist_cov=np.zeros((T, D, D, nb), np.float32),
               free_energy=np.zeros((T, nb)), status=np.zeros(nb, np.int32))
    rc = lib.multinomial_host_online(K, T, ctypes.c_longlong(nb), its, _P(_prior_block(xi0, W0)), int(start),
                                     _P(carry[0]), _P(carry[1]), _P(np.ascontiguousarray(y, np.int32)),
                                     *(_P(out[k]) for k in ("hist_mean", "hist_cov", "free_energy", "status")))
    assert rc == 0
    out["m"], out["S"] = carry
    return out


@pytest.mark.parametrize("K", [2, 3, 10, 33, 40, 64])
def test_the_kernel_bodies_on_the_host_against_the_reference(K):
    lib = _host_harness()
    for n in (1, 200):
        y, xi0, W0 = random_problem(K, n, 3, seed=100 * K + n)
        r = run_host(lib, y, xi0, W0, 10)
        gate(f"K={K} n={n}", r, reference_on_f32(y, xi0, W0, 10))
        assert (r["status"] == 0).all()
        np.testing.assert_array_equal(r["psi_mean"], r["hist_mean"][-1])
        np.testing.assert_array_equal(r["psi_cov"], r["hist_cov"][-1])
    y, xi0, W0 = random_problem(K, 25, 2, seed=7 * K)
    for its in (1, 3):
        r = run_host_online(lib, y, xi0, W0, its)
        ref = online_reference_on_f32(y, xi0, W0, its)
        gate(f"online K={K} its={its}", r, ref)
        np.testing.assert_allclose(r["m"], ref["m"], rtol=1e-10, atol=1e-12)
        np.testing.assert_allclose(r["S"], ref["S"], rtol=1e-10, atol=1e-12)


def test_online_in_chunks_is_one_call_bit_for_bit():
    lib = _host_harness()
    y, xi0, W0 = random_problem(12, 40, 3, seed=9)
    whole = run_host_online(lib, y, xi0, W0, 2)
    parts, carry = [], None
    for a, b in ((0, 1), (1, 8), (8, 9), (9, 40)):
        o = run_host_online(lib, y[a:b], xi0, W0, 2, carry)
        carry = (o["m"], o["S"])
        parts.append(o)
    for k in ("hist_mean", "hist_cov", "free_energy"):
        np.testing.assert_array_equal(np.concatenate([p[k] for p in parts]), whole[k])
    np.testing.assert_array_equal(carry[0], whole["m"])
    np.testing.assert_array_equal(carry[1], whole["S"])


def test_the_kernel_bodies_flag_negative_counts_and_read_the_sample_as_zero():
    lib = _host_harness()
    y, xi0, W0 = random_problem(4, 60, 4, seed=11)
    bad = y.copy()
    bad[3, 2, 1] = -1
    r = run_host(lib, bad, xi0, W0, 6)
    assert r["status"].tolist() == [0, 1, 0, 0]
    clean = y.copy()
    clean[3, :, 1] = 0
    gate("negative count", r, reference_on_f32(clean, xi0, W0, 6))
    o = run_host_online(lib, bad[:10], xi0, W0)
    assert o["status"].tolist() == [0, 1, 0, 0]
    gate("negative count online", o, online_reference_on_f32(clean[:10], xi0, W0))


# ---------------------------------------------------------------- argument handling of infer (before any device work)
def test_infer_refuses_what_it_cannot_run(rx):
    from rxinfer_jl_b200.distributions import MvNormalWeightedMeanPrecision
    model = rx.multinomial_regression(np.zeros(3), np.eye(3))
    y, _, _ = random_problem(4, 10, 3, seed=0)
    data = {"y": y.transpose(2, 0, 1)}
    for kw in (dict(constraints=object()), dict(predictvars=rx.KeepLast()), dict(returnvars={"ω": rx.KeepLast()}),
               dict(returnvars="ψ"), dict(initialization={"ψ": None}), dict(keephistory=10), dict(autoupdates=True),
               dict(options={"force_marginal_computation": True})):
        with pytest.raises(NotImplementedError):
            rx.infer(model=model, data=data, **kw)
    with pytest.raises(NotImplementedError):
        rx.infer(model=model, datastream=iter([]))
    with pytest.raises(KeyError):
        rx.infer(model=model, data={"x": data["y"]})
    with pytest.raises(ValueError):
        rx.infer(model=model, data={**data, "z": data["y"]})
    with pytest.raises(ValueError):
        rx.infer(model=model, data={"y": data["y"] + 0.5})
    with pytest.raises(ValueError):
        rx.infer(model=model, data={"y": data["y"][0, 0]})
    with pytest.raises(TypeError):
        rx.infer(model=model, data=data, not_an_argument=1)
    online = rx.multinomial_regression_online()
    init = {"ψ": MvNormalWeightedMeanPrecision(np.zeros(3), np.eye(3))}
    with pytest.raises(ValueError):                    # no autoupdates
        rx.infer(model=online, data=data, initialization=init)
    with pytest.raises(ValueError):                    # no initialization of ψ
        rx.infer(model=online, data=data, autoupdates=True)
    with pytest.raises(NotImplementedError):
        rx.infer(model=online, data=data, initialization=init, autoupdates=True, returnvars=rx.KeepLast())
    with pytest.raises(ValueError):
        rx.infer(model=online, data={"y": data["y"], "x": 1}, initialization=init, autoupdates=True)
    with pytest.raises(ValueError):                    # streaming needs the batch
        rx.infer(model=online, initialization=init, autoupdates=True)
