"""Bayesian binomial / logistic regression (BinomialPolya, mean-field Pólya-Gamma VMP; DESIGN 3.21), CPU only: the fp64
reference of oracle/binomial.py against the Pólya-Gamma series, the uncollapsed bound and quadrature evidence; its free
energy never increases; Bernoulli mode, n = 0 padding; the reference test's own assertions (binomialreg_tests.jl:97-106)
on the reference; the kernel body compiled for the host (tests/c/binomial_host_harness.cu) against the reference at
p = 1..8; the path selection; and the argument handling of ``infer``."""
import ctypes
import os
import shutil
import subprocess

import numpy as np
import pytest
from scipy.special import gammaln
from scipy.stats import norm

from oracle import binomial as ob
from util import TOL_COV, TOL_MEAN

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FE_TOL = 1e-5


def random_problem(p, N, nb, seed, bernoulli=False, scale=1.0):
    """X [N, p, nb], y and n [N, nb] int32 (n None in Bernoulli mode), and a prior xi0 [p], W0 [p, p]."""
    rng = np.random.default_rng(seed)
    X = (scale * rng.standard_normal((N, p, nb))).astype(np.float32)
    beta = rng.standard_normal((p, nb))
    n = np.ones((N, nb), np.int32) if bernoulli else rng.integers(0, 21, (N, nb)).astype(np.int32)
    prob = 1 / (1 + np.exp(-np.einsum("ijb,jb->ib", X.astype(np.float64), beta)))
    y = rng.binomial(n, prob).astype(np.int32)
    A = rng.standard_normal((p, p))
    W0 = A @ A.T / p + np.eye(p)
    xi0 = 0.3 * rng.standard_normal(p)
    return X, y, (None if bernoulli else n), xi0, W0


def reference_on_f32(X, y, n, xi0, W0, its, want_free_energy=True):
    """The fp64 reference on the inputs the kernel sees (the prior rounded to fp32)."""
    f32 = lambda a: np.asarray(a, np.float32).astype(np.float64)
    return ob.vmp_batch(np.asarray(X, np.float64), y, n, f32(xi0), f32(W0), its, want_free_energy)


def gate(case, r, ref, chains=None, fe=True):
    """Per chain: mean at TOL_MEAN and covariance at TOL_COV relative L2 over the iterations, F at FE_TOL relative to
    max(|F|, 1).  Returns the worst errors."""
    nb = ref["hist_mean"].shape[-1]
    worst = {}
    for b in range(nb) if chains is None else chains:
        for key, tol in (("hist_mean", TOL_MEAN), ("hist_cov", TOL_COV)):
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
def test_omega_bar_against_the_polya_gamma_series():
    c = np.array([0.0, 1e-6, 1e-4, 1e-3, 0.05, 0.5, 1.0, 3.0, 10.0, 40.0])
    k = np.arange(1, 400001)[:, None]
    for n in (1, 7, 20):
        series = n / (2 * np.pi ** 2) * (1 / ((k - 0.5) ** 2 + c[None] ** 2 / (4 * np.pi ** 2))).sum(0)
        tail = n / (2 * np.pi ** 2) / (k[-1, 0] - 0.5)          # the series' tail beyond the last term, ~ 1 / k
        np.testing.assert_allclose(ob.omega_bar(n, c), series + tail, rtol=1e-9)
    assert ob.omega_bar(4, 0.0) == 1.0


def test_the_uncollapsed_bound_is_above_the_collapsed_one_with_equality_at_c():
    X, y, n, xi0, W0 = random_problem(3, 40, 1, seed=1)
    X, y, n = X[..., 0].astype(np.float64), y[:, 0].astype(np.float64), n[:, 0].astype(np.float64)
    r = ob.vmp(X, y, n, xi0, W0, 3)
    m, S = r["mean"][-1], r["cov"][-1]
    c = np.sqrt((X @ m) ** 2 + np.einsum("ij,jk,ik->i", X, S, X))
    F = ob.free_energy(X, y, n, xi0, W0, m, S)
    np.testing.assert_allclose(ob.free_energy_uncollapsed(X, y, n, xi0, W0, m, S, c), F, rtol=1e-12)
    rng = np.random.default_rng(2)
    for _ in range(20):
        cq = c * np.exp(rng.normal(0, 0.7, c.shape)) + rng.uniform(0, 0.1, c.shape)
        assert ob.free_energy_uncollapsed(X, y, n, xi0, W0, m, S, cq) >= F - 1e-12


def _log_evidence_quadrature(X, y, n, xi0, W0):
    """log p(y) on a grid around the prior and the likelihood, p = 1 or 2."""
    p = X.shape[1]
    S0 = np.linalg.inv(W0)
    m0 = S0 @ xi0
    g = np.linspace(-8, 8, 2001 if p == 1 else 601)
    B = np.stack(np.meshgrid(*([g] * p), indexing="ij"), -1).reshape(-1, p)
    d = B - m0
    lp = -0.5 * np.einsum("ij,jk,ik->i", d, W0, d) - 0.5 * p * np.log(2 * np.pi) + 0.5 * np.linalg.slogdet(W0)[1]
    psi = B @ X.T
    ll = (gammaln(n + 1) - gammaln(y + 1) - gammaln(n - y + 1) + y * psi - n * np.logaddexp(0, psi)).sum(1)
    t = lp + ll
    return np.log(np.exp(t - t.max()).sum() * (g[1] - g[0]) ** p) + t.max()


@pytest.mark.parametrize("p", [1, 2])
def test_the_free_energy_bounds_minus_the_log_evidence(p):
    for seed in range(4):
        X, y, n, xi0, W0 = random_problem(p, 6, 1, seed=10 + seed)
        X, y, n = X[..., 0].astype(np.float64), y[:, 0].astype(np.float64), n[:, 0].astype(np.float64)
        r = ob.vmp(X, y, n, xi0, W0, 30)
        assert r["free_energy"].min() >= -_log_evidence_quadrature(X, y, n, xi0, W0) - 1e-9


def test_the_free_energy_never_increases():
    for p, seed in ((1, 0), (2, 1), (5, 2), (8, 3)):
        X, y, n, xi0, W0 = random_problem(p, 300, 3, seed=seed, scale=1.5)
        fe = reference_on_f32(X, y, n, xi0, W0, 40)["free_energy"]
        assert (np.diff(fe, axis=0) <= 1e-9 * np.maximum(np.abs(fe[1:]), 1)).all()


def test_bernoulli_mode_is_n_equal_one_and_n_zero_padding_drops_the_sample():
    X, y, _, xi0, W0 = random_problem(3, 50, 2, seed=4, bernoulli=True)
    a = reference_on_f32(X, y, None, xi0, W0, 10)
    b = reference_on_f32(X, y, np.ones_like(y), xi0, W0, 10)
    for k in ("hist_mean", "hist_cov", "free_energy"):
        np.testing.assert_array_equal(a[k], b[k])
    X, y, n, xi0, W0 = random_problem(3, 50, 2, seed=5)
    n[7], y[7] = 0, 0
    keep = np.arange(50) != 7
    a = reference_on_f32(X, y, n, xi0, W0, 10)
    b = reference_on_f32(X[keep], y[keep], n[keep], xi0, W0, 10)
    for k in ("hist_mean", "hist_cov", "free_energy"):
        np.testing.assert_allclose(a[k], b[k], rtol=1e-12, atol=1e-12)


# ---------------------------------------------------------------- the reference test (binomialreg_tests.jl:26-106)
def reference_simulations(n_sims=20, N=1000, beta=(-1.0, 0.6), seed=2024):
    """20 data sets from the reference's generating process (X ~ N(0, 1), n ~ 5..20, y ~ Binomial(n, σ(X β))) from a
    seeded numpy generator (the reference's StableRNG Binomial sampler is not restated), in the kernel layout."""
    rng = np.random.default_rng(seed)
    beta = np.asarray(beta)
    X = rng.standard_normal((N, len(beta), n_sims))
    n = rng.integers(5, 21, (N, n_sims))
    y = rng.binomial(n, 1 / (1 + np.exp(-np.einsum("ijb,j->ib", X, beta))))
    return X.astype(np.float32), y.astype(np.int32), n.astype(np.int32), beta


def reference_assertions(mean, var, fes, beta):
    """fes[end] < fes[1] per simulation; 95 % interval coverage >= 0.8 per coordinate.  mean, var [p, sims],
    fes [its, sims]."""
    assert (fes[-1] < fes[0]).all()
    u = norm.cdf(beta[:, None], loc=mean, scale=np.sqrt(var))
    coverage = ((u >= 0.025) & (u <= 0.975)).mean(1)
    assert (coverage >= 0.8).all(), coverage
    return coverage


def test_the_reference_assertions_on_the_fp64_reference():
    X, y, n, beta = reference_simulations()
    r = ob.vmp_batch(X.astype(np.float64), y, n, np.zeros(2), np.eye(2), 100)
    cov = r["hist_cov"][-1]
    reference_assertions(r["hist_mean"][-1], np.stack([cov[0, 0], cov[1, 1]]), r["free_energy"], beta)


# ---------------------------------------------------------------- the kernel body on the host
def _host_harness():
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    so = os.path.join(ROOT, "tests", "c", "_binomial_host.so")
    src = os.path.join(ROOT, "tests", "c", "binomial_host_harness.cu")
    hdrs = [os.path.join(ROOT, "rxinfer.jl_b200", "csrc", h) for h in ("rxg_polya.cuh", "rxg_normal_wishart.cuh")]
    if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(f) for f in [src] + hdrs):
        subprocess.run([nvcc, "-O2", "-Wno-deprecated-gpu-targets", "-shared", "-Xcompiler", "-fPIC", "-o", so, src], check=True)
    return ctypes.CDLL(so)


def run_host(lib, X, y, n, xi0, W0, its):
    N, p, nb = X.shape
    xi0 = np.asarray(xi0, np.float32).astype(np.float64)
    W0 = np.asarray(W0, np.float32).astype(np.float64)
    S0 = np.linalg.inv(W0)
    m0 = S0 @ xi0
    z = lambda *s: np.zeros(s, np.float32)
    out = dict(beta_mean=z(p, nb), beta_cov=z(p, p, nb), free_energy=np.zeros((its, nb)), hist_mean=z(its, p, nb),
               hist_cov=z(its, p, p, nb), status=np.zeros(nb, np.int32))
    P = lambda a: None if a is None else a.ctypes.data_as(ctypes.c_void_p)
    c = lambda a: None if a is None else np.ascontiguousarray(a)
    X, y, n = c(np.asarray(X, np.float32)), c(np.asarray(y, np.int32)), c(None if n is None else np.asarray(n, np.int32))
    rc = lib.binomial_host_run(p, N, ctypes.c_longlong(nb), its, P(c(xi0)), P(c(W0)), P(c(m0)), P(c(S0)),
                               ctypes.c_double(np.linalg.slogdet(W0)[1]), ctypes.c_double(xi0 @ m0), P(X), P(y), P(n),
                               *(P(out[k]) for k in ("beta_mean", "beta_cov", "free_energy", "hist_mean", "hist_cov",
                                                     "status")))
    assert rc == 0
    return out


@pytest.mark.parametrize("p", range(1, 9))
def test_the_kernel_body_on_the_host_against_the_reference(p):
    lib = _host_harness()
    for N, bern in ((1, False), (7, True), (400, False), (400, True)):
        X, y, n, xi0, W0 = random_problem(p, N, 3, seed=100 * p + N + bern, bernoulli=bern)
        r = run_host(lib, X, y, n, xi0, W0, 12)
        gate(f"p={p} N={N} bernoulli={bern}", r, reference_on_f32(X, y, n, xi0, W0, 12))
        assert (r["status"] == 0).all()
        np.testing.assert_array_equal(r["beta_mean"], r["hist_mean"][-1])
        np.testing.assert_array_equal(r["beta_cov"], r["hist_cov"][-1])


def test_the_kernel_body_flags_bad_samples_and_reads_them_as_n_zero():
    lib = _host_harness()
    X, y, n, xi0, W0 = random_problem(2, 60, 4, seed=7)
    y[3, 1] = n[3, 1] + 1                     # y > n
    X[5, 0, 2] = np.nan
    r = run_host(lib, X, y, n, xi0, W0, 8)
    assert r["status"].tolist() == [0, 1, 1, 0]
    n2 = n.copy()
    n2[3, 1], n2[5, 2] = 0, 0
    X2, y2 = np.nan_to_num(X), np.minimum(y, n2)
    gate("bad samples", r, reference_on_f32(X2, y2, n2, xi0, W0, 8))


def test_path_selection_follows_its_rule():
    lib = _host_harness()
    lib.binomial_select_path.restype = ctypes.c_int
    per_sm = lib.binomial_group_chains_per_sm()
    min_n = lib.binomial_group_min_n()
    for sm in (1, 78, 132):
        for batch in (1, 20, 1024, per_sm * sm, per_sm * sm + 1, 16384, 65536, 1 << 20):
            for N in (1, min_n - 1, min_n, 1000, 10000):
                for p in (1, 2, 8):
                    want = 2 if (batch <= per_sm * sm and N >= min_n) else 1
                    assert lib.binomial_select_path(ctypes.c_longlong(batch), N, p, sm) == want, (batch, N, p, sm)


# ---------------------------------------------------------------- argument handling of infer (before any device work)
def test_infer_refuses_what_it_cannot_run(rx):
    model = rx.binomial_regression(np.zeros(2), np.eye(2))
    X, y, n, _, _ = random_problem(2, 10, 3, seed=0)
    data = {"X": X.transpose(2, 0, 1), "y": y.T, "n_trials": n.T}
    with pytest.raises(NotImplementedError):
        rx.infer(model=model, data=data, constraints=object())
    with pytest.raises(NotImplementedError):
        rx.infer(model=model, data=data, predictvars=rx.KeepLast())
    with pytest.raises(NotImplementedError):
        rx.infer(model=model, data=data, returnvars={"ω": rx.KeepLast()})
    with pytest.raises(NotImplementedError):
        rx.infer(model=model, data=data, returnvars="β")
    with pytest.raises(NotImplementedError):
        rx.infer(model=model, data=data, initialization={"β": None})
    with pytest.raises(NotImplementedError):
        rx.infer(model=model, data=data, keephistory=10)
    with pytest.raises(NotImplementedError):
        rx.infer(model=model, datastream=iter([]))
    with pytest.raises(NotImplementedError):
        rx.infer(model=model, data=data, options={"force_marginal_computation": True})
    with pytest.raises(KeyError):
        rx.infer(model=model, data={"X": data["X"]})
    with pytest.raises(ValueError):
        rx.infer(model=model, data={**data, "z": data["y"]})
    with pytest.raises(ValueError):
        rx.infer(model=model, data={**data, "y": data["y"][:, :5]})
    with pytest.raises(ValueError):
        rx.infer(model=model, data={**data, "n_trials": data["n_trials"] + 0.5})
    with pytest.raises(ValueError):
        rx.infer(model=model, data={**data, "X": data["X"][0, 0]})
    with pytest.raises(TypeError):
        rx.infer(model=model, data=data, not_an_argument=1)
