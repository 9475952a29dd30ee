"""Gamma mixture model with point-mass shapes (DESIGN 3.24), CPU half: the fp64 reference (oracle/gamma_mixture.py) against
the definition of its free energy and of each update, the point-mass shape as the maximiser, F non-increasing under every
update order, statistical recovery, the kernel body compiled for the host (tests/c/gamma_mixture_host_harness.cu) against
the reference, the replay of the reference test's data and its assertions, and the argument handling of ``infer``."""
import ctypes
import itertools
import os
import shutil
import subprocess

import numpy as np
import pytest
from scipy import integrate, stats
from scipy.special import digamma, gammaln

from oracle import gamma_mixture as og

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KEYS = ("alpha_s", "a_shape0", "a_rate0", "b_shape0", "b_rate0", "alpha_init", "b_shape_init", "b_rate_init", "a_start")
BLOCKS = ("a_shape0", "a_rate0", "b_shape0", "b_rate0", "alpha_s", "alpha_init", "b_shape_init", "b_rate_init", "a_start")


def f32(x):
    return np.asarray(x, np.float32).astype(np.float64)


def problem(K, N, batch, seed, overlap=False):
    """Distinct data per chain from K Gamma components (means spread over a decade, or all near 1 with ``overlap``) and
    hyper-parameters drawn around them."""
    rng = np.random.default_rng(seed)
    shapes = rng.uniform(2.0, 40.0, K)
    means = np.full(K, 1.0) * rng.uniform(0.8, 1.2, K) if overlap else np.geomspace(0.2, 5.0, K) * rng.uniform(0.9, 1.1, K)
    w = rng.dirichlet(np.full(K, 3.0))
    y = np.empty((N, batch))
    for b in range(batch):
        z = rng.choice(K, N, p=w)
        y[:, b] = rng.gamma(shapes[z], means[z] / shapes[z]) * rng.uniform(0.8, 1.25)
    pri = dict(alpha_s=rng.uniform(0.5, 5.0, K), a_shape0=rng.uniform(1.0, 3.0, K), a_rate0=rng.uniform(0.01, 0.5, K),
               b_shape0=rng.uniform(0.5, 5.0, K), b_rate0=rng.uniform(0.2, 3.0, K) * shapes / means / 10,
               alpha_init=rng.uniform(0.5, 5.0, K), b_shape_init=rng.uniform(0.5, 3.0, K),
               b_rate_init=rng.uniform(0.5, 3.0, K), a_start=rng.uniform(0.5, 3.0, K))
    return y, pri


# --------------------------------------------------------------------------- the free energy against its definition
def dense_free_energy(y, r, alpha, a, bsh, brt, pri):
    """F = E_q[log q] - E_q[log p] with the entropies of scipy's distributions and every expectation integrated
    numerically: E[log s_k] over the Beta marginal of q(s), E[b] and E[log b] over q(b_k)."""
    K = len(a)
    el = lambda f, dist: integrate.quad(lambda x: f(x) * dist.pdf(x), 0, np.inf if dist.dist.name == "gamma" else 1,
                                        epsabs=1e-14, epsrel=1e-13, limit=200)[0]
    qs = [stats.beta(alpha[k], alpha.sum() - alpha[k]) for k in range(K)]
    qb = [stats.gamma(bsh[k], scale=1.0 / brt[k]) for k in range(K)]
    els = np.array([el(np.log, q) for q in qs])
    elb = np.array([el(np.log, q) for q in qb])
    eb = np.array([el(lambda x: x, q) for q in qb])
    a0 = np.asarray(pri["alpha_s"], np.float64)
    logp_s = gammaln(a0.sum()) - gammaln(a0).sum() + ((a0 - 1) * els).sum()
    F = -stats.dirichlet(alpha).entropy() - logp_s
    for k in range(K):
        bs0, br0 = pri["b_shape0"][k], pri["b_rate0"][k]
        F -= qb[k].entropy() + bs0 * np.log(br0) - gammaln(bs0) + (bs0 - 1) * elb[k] - br0 * eb[k]
        F -= stats.gamma(pri["a_shape0"][k], scale=1.0 / pri["a_rate0"][k]).logpdf(a[k])
    for i in range(len(y)):
        ll = els + a * elb - gammaln(a) + (a - 1) * np.log(y[i]) - eb * y[i]
        F -= (r[i] * ll).sum() - (r[i] * np.log(r[i])).sum()
    return F


@pytest.mark.parametrize("K", [2, 3, 8])
def test_closed_form_free_energy_equals_the_definition(K):
    y, pri = problem(K, 30, 1, seed=K)
    rng = np.random.default_rng(10 + K)
    r = rng.dirichlet(np.ones(K), 30)
    alpha, a = rng.uniform(1.5, 20.0, K), rng.uniform(0.5, 30.0, K)
    bsh, brt = rng.uniform(1.5, 50.0, K), rng.uniform(0.5, 50.0, K)
    got = og.free_energy(y, r[:, :, None], alpha[:, None], a[:, None], bsh[:, None], brt[:, None], pri)[0]
    want = dense_free_energy(y[:, 0], r, alpha, a, bsh, brt, pri)
    assert abs(got - want) < 1e-10 * max(abs(want), 1.0), (got, want)


# --------------------------------------------------------------------------- the updates
@pytest.mark.parametrize("K", [2, 3, 8])
def test_every_update_is_the_conjugate_update_from_sufficient_statistics(K):
    """Each update as the product of its prior and the per-datum messages of the uniform initial q(z): q(b_k) = prior x
    prod_i Gamma(1 + â r_ik, r_ik y_i) (shape / rate), q(s) = prior x prod_i Dirichlet(1 + r_i); q(z_i) from E[log s] and
    E[log Gamma(y_i | â, b)] integrated over q(b); â from the statistics (gradient zero)."""
    y, pri = problem(K, 40, 2, seed=20 + K)
    N = len(y)
    r = 1.0 / K
    run = lambda sch: og.gamma_mixture(y, **pri, iterations=1, schedule=sch)
    a0 = np.asarray(pri["a_start"])[:, None]
    res = run("bazs")                 # q(b) first: from â = a_start
    want_sh = np.asarray(pri["b_shape0"])[:, None] + sum(a0 * r for _ in range(N))
    want_rt = np.asarray(pri["b_rate0"])[:, None] + sum(r * y[i] for i in range(N))[None]
    np.testing.assert_allclose(res["hist_b_shape"][0], np.broadcast_to(want_sh, (K, 2)), rtol=1e-13)
    np.testing.assert_allclose(res["hist_b_rate"][0], want_rt, rtol=1e-13)
    res = run("sabz")
    np.testing.assert_allclose(res["alpha"], np.asarray(pri["alpha_s"])[:, None] + np.full((K, 2), N * r), rtol=1e-13)
    res = run("zabs")                 # q(z) first: from q(s) = alpha_init, â = a_start, q(b) = the initial one
    ai = np.asarray(pri["alpha_init"])
    for b in range(2):
        for i in (0, N - 1):
            lr = []
            for k in range(K):
                qb = stats.gamma(pri["b_shape_init"][k], scale=1.0 / pri["b_rate_init"][k])
                ell = qb.expect(lambda x: stats.gamma(pri["a_start"][k], scale=1.0 / x).logpdf(y[i, b]), epsabs=1e-13,
                                epsrel=1e-12)
                lr.append(digamma(ai[k]) - digamma(ai.sum()) + ell)
            p = np.exp(np.array(lr) - max(lr))
            np.testing.assert_allclose(res["z_prob"][i, :, b], p / p.sum(), rtol=1e-9, atol=1e-12)
    res = run("absz")                 # â first: from the uniform q(z) and the initial q(b)
    Nk, Lk = np.full(K, N * r), r * np.log(y).sum(0)
    for b in range(2):
        elb = digamma(np.asarray(pri["b_shape_init"])) - np.log(pri["b_rate_init"])
        a = res["hist_a"][0, :, b]
        g = (np.asarray(pri["a_shape0"]) - 1) / a - pri["a_rate0"] + Nk * elb + Lk[b] - Nk * digamma(a)
        assert np.abs(g).max() < 1e-9 * (np.abs(Nk * elb).max() + np.abs(Lk[b]) + 1)


def shape_objective(a, ash, art, n, c):
    return (ash - 1) * np.log(a) - art * a + a * c - n * gammaln(a)


@pytest.mark.parametrize("ash,art,n,c", [(1.0, 10.0, 200.0, 200 * 0.6), (1.0, 1.0, 50.0, 50 * 4.2), (2.5, 0.3, 3.0, -1.0),
                                         (1.0, 0.1, 1e-3, -0.05), (1.0, 1.0, 250.0, 250 * 7.0), (4.0, 2.0, 0.5, 3.0)])
def test_the_point_mass_is_the_maximiser_and_does_not_depend_on_the_start(ash, art, n, c):
    a, ok = og.point_mass_shape(ash, art, n, c, 1.0)
    assert ok and a > 0
    h = 1e-6 * a
    grad = (shape_objective(a + h, ash, art, n, c) - shape_objective(a - h, ash, art, n, c)) / (2 * h)
    scale = abs(c) + art + n * abs(digamma(a)) + (ash - 1) / a
    assert abs(grad) < 1e-5 * scale, grad
    grid = a * np.exp(np.linspace(-3, 3, 2001))
    assert (shape_objective(grid, ash, art, n, c) <= shape_objective(a, ash, art, n, c) + 1e-12 * scale).all()
    for start in (1e-4, 0.3, 7.0, 1e3, 1e6):
        a2, ok2 = og.point_mass_shape(ash, art, n, c, start)
        assert ok2 and abs(a2 - a) <= 1e-10 * a, (start, a2, a)


def test_a_shape_objective_without_a_maximiser_is_not_converged():
    """N_k = 0 with a shape prior of 1: f(a) = -rate a + const has its supremum at a -> 0, which Newton cannot reach."""
    _, ok = og.point_mass_shape(1.0, 1.0, 0.0, 0.0, 1.0)
    assert not ok


@pytest.mark.parametrize("K,overlap", [(2, False), (3, True), (5, False)])
def test_free_energy_never_increases_under_any_update_order(K, overlap):
    y, pri = problem(K, 60, 3, seed=30 + K, overlap=overlap)
    for sch in itertools.permutations("absz"):
        fe = og.gamma_mixture(y, **pri, iterations=15, schedule="".join(sch))["free_energy"]
        assert (np.diff(fe, axis=0) <= 1e-9 * np.maximum(np.abs(fe[1:]), 1.0)).all(), sch


def test_statistical_recovery_of_two_separated_components():
    """5 000 draws from Gamma(shape 4, rate 8) (mean 0.5) and Gamma(shape 30, rate 10) (mean 3), weights 0.6 / 0.4, fitted
    from vague priors with the initial q(b) breaking the symmetry: the fitted shapes within 10 %, the component means
    within 2 % and the weights within 0.02 of the truth."""
    rng = np.random.default_rng(2024)
    n = 5000
    z = rng.random(n) < 0.6
    y = np.where(z, rng.gamma(4.0, 1 / 8.0, n), rng.gamma(30.0, 1 / 10.0, n))[:, None]
    pri = dict(alpha_s=[1.0, 1.0], a_shape0=[1.0, 1.0], a_rate0=[0.01, 0.01], b_shape0=[1.0, 1.0], b_rate0=[0.1, 0.1],
               alpha_init=[1.0, 1.0], b_shape_init=[1.0, 10.0], b_rate_init=[1.0, 1.0], a_start=[1.0, 1.0])
    r = og.gamma_mixture(y, **pri, iterations=400)
    a = r["a_hat"][:, 0]
    means = a / (r["b_shape"] / r["b_rate"])[:, 0]
    w = r["alpha"][:, 0] / r["alpha"][:, 0].sum()
    assert r["converged"].all()
    np.testing.assert_allclose(a, [4.0, 30.0], rtol=0.10)
    np.testing.assert_allclose(means, [0.5, 3.0], rtol=0.02)
    np.testing.assert_allclose(w, [0.6, 0.4], atol=0.02)


# --------------------------------------------------------------------------- the kernel body on the host
def _host_harness():
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    so = os.path.join(ROOT, "tests", "c", "_gamma_mixture_host.so")
    src = os.path.join(ROOT, "tests", "c", "gamma_mixture_host_harness.cu")
    hdrs = [os.path.join(ROOT, "rxinfer.jl_b200", "csrc", h) for h in ("rxg_gamma_mixture.cuh", "rxg_hmm.cuh")]
    if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(f) for f in [src] + hdrs):
        subprocess.run([nvcc, "-O2", "-Wno-deprecated-gpu-targets", "-shared", "-Xcompiler", "-fPIC", "-o", so, src],
                       check=True)
    lib = ctypes.CDLL(so)
    lib.gamma_mixture_trigamma.restype = ctypes.c_double
    lib.gamma_mixture_trigamma.argtypes = [ctypes.c_double]
    return lib


def params_block(pri):
    """The fp64 constant block of the C entry from fp32-rounded hyper-parameters."""
    K = len(pri["alpha_s"])
    blk = np.concatenate([f32(pri[k]) for k in BLOCKS])
    a = f32(pri["alpha_s"])
    return np.concatenate([blk, [a.sum(), gammaln(a.sum()) - gammaln(a).sum()]]), K


def run_host(lib, y, pri, its):
    prm, K = params_block(pri)
    N, nb = y.shape
    z = lambda *s: np.zeros(s, np.float32)
    out = dict(alpha=z(K, nb), a_hat=z(K, nb), b_shape=z(K, nb), b_rate=z(K, nb), free_energy=np.zeros((its, nb)),
               z_prob=z(N, K, nb), hist_a=z(its, K, nb), hist_b_shape=z(its, K, nb), hist_b_rate=z(its, K, nb),
               status=np.zeros(nb, np.int32))
    P = lambda a: a.ctypes.data_as(ctypes.c_void_p)
    y32 = np.ascontiguousarray(y, np.float32)
    rc = lib.gamma_mixture_host_run(K, N, ctypes.c_longlong(nb), its, P(prm), P(y32),
                                    *(P(out[k]) for k in ("alpha", "a_hat", "b_shape", "b_rate", "free_energy", "z_prob",
                                                          "hist_a", "hist_b_shape", "hist_b_rate", "status")))
    assert rc == 0
    return out


def reference_on_f32(y, pri, its):
    return og.gamma_mixture(f32(y), **{k: f32(v) for k, v in pri.items()}, iterations=its)


TOL_PARAM = 1e-5      # relative L2 per chain over the components: a_hat, q(b), q(s)
TOL_HIST = 3e-5       # the same over every iteration of the KeepEach histories
TOL_FE = 1e-5         # relative to max(|F|, 1), per chain: the last iteration; 3 TOL_FE for the earlier ones
TOL_Z = 1e-3          # q(z), absolute


def gate(case, got, ref):
    for k, tol in (("alpha", TOL_PARAM), ("a_hat", TOL_PARAM), ("b_shape", TOL_PARAM), ("b_rate", TOL_PARAM),
                   ("hist_a", TOL_HIST), ("hist_b_shape", TOL_HIST), ("hist_b_rate", TOL_HIST)):
        g = np.asarray(got[k], np.float64)
        ax = tuple(range(g.ndim - 1))
        err = np.sqrt(((g - ref[k]) ** 2).sum(ax)) / np.sqrt((ref[k] ** 2).sum(ax))
        assert err.max() < tol, f"{case}: {k} worst chain {int(err.argmax())} err {err.max():.3g} > {tol}"
    efe = np.abs(np.asarray(got["free_energy"]) - ref["free_energy"]) / np.maximum(np.abs(ref["free_energy"]), 1.0)
    assert efe[-1].max() < TOL_FE, f"{case}: last free energy {efe[-1].max():.3g}"
    assert efe.max() < 3 * TOL_FE, f"{case}: free energy history {efe.max():.3g}"
    ez = np.abs(np.asarray(got["z_prob"], np.float64) - ref["z_prob"]).max()
    assert ez < TOL_Z, f"{case}: z_prob {ez:.3g}"


def test_trigamma_of_the_kernel():
    from scipy.special import polygamma
    lib = _host_harness()
    for x in (1e-6, 0.01, 0.5, 1.0, 3.3, 9.99, 10.0, 57.0, 1e4, 1e9):
        assert abs(lib.gamma_mixture_trigamma(x) - polygamma(1, x)) <= 1e-14 * polygamma(1, x), x


@pytest.mark.parametrize("K", [2, 3, 8])
def test_the_kernel_body_on_the_host_against_the_reference(K):
    lib = _host_harness()
    for N, its, overlap in ((1, 1, False), (7, 50, True), (250, 1, True), (250, 50, False)):
        y, pri = problem(K, N, 5, seed=100 * K + N + its, overlap=overlap)
        ref = reference_on_f32(y, pri, its)
        got = run_host(lib, y, pri, its)
        assert (got["status"] == 0).all() and ref["converged"].all()
        gate(f"K={K} N={N} its={its} overlap={overlap}", got, ref)
        np.testing.assert_array_equal(got["a_hat"], got["hist_a"][-1])
        np.testing.assert_array_equal(got["b_rate"], got["hist_b_rate"][-1])


def test_the_kernel_body_flags_bad_data_with_nan_outputs():
    lib = _host_harness()
    y, pri = problem(3, 40, 4, seed=9)
    y[5, 1], y[7, 2] = 0.0, np.inf
    got = run_host(lib, y, pri, 6)
    assert got["status"].tolist() == [0, 1, 1, 0]
    for k, v in got.items():
        if k != "status":
            assert np.isnan(v[..., [1, 2]]).all() and np.isfinite(v[..., [0, 3]]).all(), k
    ref = reference_on_f32(y[:, [0, 3]], pri, 6)
    gate("bad data", {k: v[..., [0, 3]] for k, v in got.items()}, ref)


# --------------------------------------------------------------------------- the reference test's data
def gamma_mt(rng, shape, scale):
    """Distributions' GammaMTSampler (Marsaglia & Tsang 2000) as read here: d = shape - 1/3, c = 1 / (3 sqrt(d)); draw
    x = randn until v = (1 + c x)^3 > 0, u = rand; accept on the squeeze u < 1 - 0.0331 x^4 or on log u < x^2 / 2 +
    d (1 - v + log v); return d v scale."""
    d = shape - 1.0 / 3.0
    c = 1.0 / (3.0 * np.sqrt(d))
    while True:
        x = rng.randn()
        cv = 1.0 + c * x
        while cv <= 0.0:
            x = rng.randn()
            cv = 1.0 + c * x
        v = cv ** 3
        u = rng.rand()
        if u < 1.0 - 0.0331 * x ** 4 or np.log(u) < 0.5 * x * x + d * (1.0 - v + np.log(v)):
            return d * v * scale


def reference_data(reading=None):
    """gamma_mixture_tests.jl:45-57: StableRNG(43); mixing = rand(rng, 2) normalised; 250 draws of MixtureModel([Gamma(9,
    1/27), Gamma(90, 1/270)], mixing), each a label (Categorical, ``reading`` of test_mixture.CATEGORICAL_READINGS) and
    then the component's Gamma draw."""
    from oracle.julia_rng import StableRNG
    from test_mixture import CATEGORICAL_READINGS, DEFAULT_READING
    rng = StableRNG(43)
    mixing = np.array([rng.rand(), rng.rand()])
    mixing /= mixing.sum()
    comps = [(9.0, 1.0 / 27.0), (90.0, 1.0 / 270.0)]
    draw = CATEGORICAL_READINGS[reading or DEFAULT_READING]
    y = np.array([gamma_mt(rng, *comps[draw(rng, list(mixing), 1)[0] - 1]) for _ in range(250)])
    return y, mixing


def reference_model(mixing):
    """gamma_mixture_tests.jl:59-71 through infer's objects: Distributions' Gamma(shape, scale) priors as shape / rate."""
    from rxinfer_jl_b200 import Categorical, Dirichlet, GammaShapeRate, vague
    from rxinfer_jl_b200.inference import GammaMixtureConstraints, gamma_mixture
    model = gamma_mixture(K=2, prior_s=Dirichlet(1e3 * mixing),
                          priors_as=[GammaShapeRate(1.0, 1 / 0.1), GammaShapeRate(1.0, 1.0)],
                          priors_bs=[GammaShapeRate(10.0, 1 / 2.0), GammaShapeRate(1.0, 1 / 3.0)])
    init = {"s": Dirichlet(1e3 * mixing), "z": vague(Categorical, 2), "bs": GammaShapeRate(1.0, 1.0)}
    return model, GammaMixtureConstraints(a_start=1.0), init


def reference_arrays(mixing):
    from rxinfer_jl_b200.inference import gamma_mixture_arguments
    return gamma_mixture_arguments(*reference_model(mixing))


def reference_assertions(a_hat, b_mean, s_mean):
    """gamma_mixture_tests.jl:90-94 without the free-energy pin, which no data reading reproduces (DESIGN 3.24)."""
    means = np.asarray(a_hat) / np.asarray(b_mean)
    assert abs(means[0] - 0.32) <= 1e-2 and abs(means[1] - 0.33) <= 1e-2, means
    np.testing.assert_allclose(s_mean, [0.8, 0.2], atol=1e-2)


def test_the_mixing_weights_are_replayed():
    _, mixing = reference_data()
    np.testing.assert_allclose(mixing, [0.79991, 0.20009], atol=1e-5)


@pytest.mark.parametrize("schedule", ["absz", "zabs", "bazs"])
def test_the_reference_assertions_on_the_fp64_reference(schedule):
    from test_mixture import CATEGORICAL_READINGS
    for reading in CATEGORICAL_READINGS:
        y, mixing = reference_data(reading)
        arr = reference_arrays(mixing)
        r = og.gamma_mixture(y[:, None], **arr, iterations=50, schedule=schedule)
        assert r["converged"].all()
        reference_assertions(r["a_hat"][:, 0], (r["b_shape"] / r["b_rate"])[:, 0], (r["alpha"] / r["alpha"].sum(0))[:, 0])
        assert -144.0 < r["free_energy"][-1, 0] < -138.0          # the pin is -146.8 +- 0.2 (DESIGN 3.24)


# --------------------------------------------------------------------------- infer
def test_infer_argument_handling_and_refusals(rx):
    from rxinfer_jl_b200 import Categorical, Dirichlet, GammaShapeRate
    from rxinfer_jl_b200.inference import GammaMixtureConstraints, MeanField, gamma_mixture_arguments
    y, mixing = reference_data()
    model, cons, init = reference_model(mixing)
    arr = gamma_mixture_arguments(model, cons, init)
    np.testing.assert_allclose(arr["a_rate0"], [10.0, 1.0])
    np.testing.assert_allclose(arr["b_rate0"], [0.5, 1 / 3])
    np.testing.assert_allclose(arr["b_shape_init"], [1.0, 1.0])
    np.testing.assert_allclose(arr["a_start"], [1.0, 1.0])
    a2 = gamma_mixture_arguments(model, GammaMixtureConstraints(a_start=[2.0, 3.0]),
                                 dict(init, bs=[GammaShapeRate(1.0, 2.0), GammaShapeRate(3.0, 4.0)]))
    np.testing.assert_allclose(a2["a_start"], [2.0, 3.0])
    np.testing.assert_allclose(a2["b_rate_init"], [2.0, 4.0])
    data = {"y": y}
    run = lambda **kw: rx.infer(**{**dict(model=model, data=data, constraints=cons, initialization=init,
                                          iterations=3), **kw})
    # factorisations other than the point-mass one
    for bad in (MeanField(), None, object()):
        with pytest.raises(ValueError, match="no conjugate posterior"):
            run(constraints=bad)
    # streaming keywords, predictions, datastream
    for kw in (dict(keephistory=10), dict(autoupdates=object()), dict(batch=4), dict(historyvars={}),
               dict(predictvars=rx.KeepLast()), dict(datastream=iter([]), data=None)):
        with pytest.raises(NotImplementedError):
            run(**kw)
    # returnvars: KeepEach for as / bs only
    with pytest.raises(NotImplementedError, match="KeepLast"):
        run(returnvars={"s": rx.KeepEach()})
    with pytest.raises(NotImplementedError):
        run(returnvars={"w": rx.KeepLast()})
    # initialization
    with pytest.raises(NotImplementedError, match="uniform"):
        run(initialization=dict(init, z=Categorical(np.array([0.9, 0.1]))))
    with pytest.raises(ValueError):
        run(initialization={"s": init["s"]})
    with pytest.raises(ValueError):
        run(initialization=dict(init, a=GammaShapeRate(1.0, 1.0)))
    with pytest.raises(TypeError):
        run(initialization=dict(init, s=GammaShapeRate(1.0, 1.0)))
    with pytest.raises(ValueError):
        run(initialization=dict(init, bs=[GammaShapeRate(1.0, 1.0)] * 3))
    # the model
    with pytest.raises(NotImplementedError, match=">= 1"):
        run(model=type(model)(K=2, prior_s=model.prior_s, priors_as=[GammaShapeRate(0.5, 1.0)] * 2,
                              priors_bs=model.priors_bs))
    with pytest.raises(NotImplementedError):
        run(model=type(model)(K=9, prior_s=Dirichlet(np.ones(9)), priors_as=[GammaShapeRate(1.0, 1.0)] * 9,
                              priors_bs=[GammaShapeRate(1.0, 1.0)] * 9), initialization=dict(init, s=Dirichlet(np.ones(9))))
    with pytest.raises(ValueError):
        run(model=type(model)(K=2, prior_s=model.prior_s, priors_as=model.priors_as,
                              priors_bs=[GammaShapeRate(1.0, 0.0)] * 2))
    with pytest.raises(ValueError):
        run(constraints=GammaMixtureConstraints(a_start=-1.0))
    with pytest.raises(ValueError):
        run(constraints=GammaMixtureConstraints(a_start=[1.0, 2.0, 3.0]))
    # data
    with pytest.raises(KeyError):
        run(data={"x": y})
    with pytest.raises(ValueError):
        run(data={"y": y, "u": y})
    with pytest.raises(ValueError):
        run(data={"y": np.ones((3, 4, 5))})
    with pytest.raises(NotImplementedError):
        run(meta={})
