"""``infer()``: the entry point of the reference (/root/reference/src/inference/inference.jl:577-733)
mirrored for the batched Gaussian hot path.

In the reference ``infer`` builds a factor graph from an ``@model`` and lets ReactiveMP/Rocket
schedule one message at a time (src/inference/batch.jl:103-482, streaming.jl:536-845).  Here the
``model`` argument is the *recognised pattern* -- what the Julia-side shim (julia/RxGaussB200.jl)
extracts from the GraphPPL graph -- and ``data`` carries ``batch`` independent series at once.
The keyword surface, the result object and the error behaviour follow the reference; every
keyword that would need machinery outside the hot path raises ``NotImplementedError`` instead of
being silently ignored (SURVEY.md appendix C: those calls must be routed to stock ReactiveMP).
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import NamedTuple

import numpy as np
import torch

from . import _lib as L
from .context import Context
from .distributions import (Beta, Categorical, Dirichlet, DirichletCollection, GammaShapeRate, MvNormalMeanCovariance,
                            MvNormalWeightedMeanPrecision, NormalMeanVariance, PointMass, Wishart, WishartFast)


# --------------------------------------------------------------------------- recognised models
@dataclass
class linear_gaussian_ssm_smoothing:
    """``@model linear_gaussian_ssm_smoothing(y, A, B, P, Q)``
    (/root/reference/benchmarks/Linear Multivariate Gaussian State Space Model Benchmark.ipynb:95-105;
    same graph as test/models/statespace/mlgssm_test.jl:8-17 with the prior on x[1]).
    ``x0 = (mean, cov)`` of the prior on x[1]."""
    A: np.ndarray
    B: np.ndarray
    P: np.ndarray
    Q: np.ndarray
    x0: tuple
    per_chain: bool = False     # model matrices carry a trailing [batch] axis (CUDA tensors)
    u: object = None            # constant offset: x[t] ~ MvNormal(A x[t-1] + u, P)  (`+` with a PointMass)
    prior_on_previous_state: bool = False   # x_prior ~ x0; x[1] ~ N(A x_prior + u, P)  (mlgssm_test.jl:8-17)
    horizon: int = 0            # forecast steps x[T+1..T+H], o[1..H] ~ N(B x[T+k], Q) (model_1, prediction_tests.jl:197-213)


@dataclass
class linear_gaussian_ssm_filtering(linear_gaussian_ssm_smoothing):
    """One-step model + ``@autoupdates x_min_t_mean, x_min_t_cov = mean_cov(q(x_t))``
    (ipynb:107-113, 199-216): the prior is pushed through (A, P) before every datum."""


@dataclass
class hgf:
    """``@model hgf`` with ``hgfconstraints`` / ``hgfmeta`` / autoupdates of
    /root/reference/test/models/statespace/hgf_tests.jl:10-69."""
    real_k: float = 1.0
    real_w: float = 0.0
    z_variance: float = 0.2 ** 2
    y_variance: float = 0.1 ** 2
    init: tuple = (0.0, 5.0, 0.0, 5.0)      # q(zt) = N(0,5), q(xt) = N(0,5)  (hgf_tests.jl:51-54)


@dataclass
class univariate_lgssm_gamma_precision:
    """Scalar random walk observed with unknown precision tau ~ Gamma(a0, b0), q(x) q(tau)
    (rules of /root/reference/test/models/aliases/aliases_gamma_tests.jl; SURVEY.md 8f rank 3)."""
    a: float = 1.0
    v_proc: float = 1.0
    x0: tuple = (0.0, 100.0)
    gamma_prior: tuple = (1.0, 1.0)
    init_E_tau: float = 1.0


@dataclass
class kalman_gamma_streaming:
    """The reference's ``test_model1`` (/root/reference/test/inference/inference_tests.jl:752-775): one-step random
    walk observed with unknown precision, ``constraints = MeanField()``, ``@autoupdates`` of ``mean_var(q(x_t))`` and
    ``shape / rate of q(τ)``; ``init = (m_x, v_x, shape, rate)`` of the ``@initialization`` (:766-769)."""
    transition_precision: float = 1.0
    init: tuple = (0.0, 1e3, 1.0, 1.0)


@dataclass
class latent_autoregressive:
    """``lar_model`` with ``lar_constraints`` / ``lar_init_marginals``
    (/root/reference/test/models/autoregressive/lar_tests.jl:52-122): gamma ~ Gamma, theta ~ N(0, I / w0), x0 ~ N(0, I / p0),
    x[t] ~ AR(x[t-1], theta, gamma) with ARMeta(variate, order, ARsafe()), y[t] ~ Normal(dot(c, x[t]), 1 / tau), c = e1,
    q(x, x0) q(gamma) q(theta).  The Univariate case is order = 1."""
    order: int
    tau: float
    gamma_prior: tuple = (1.0, 1.0)
    theta_prior_precision: float = 1.0
    x0_prior_precision: float = 1.0
    init_gamma: tuple = (1.0, 1.0)          # q(gamma) of the @initialization
    init_theta_precision: float = 1.0       # q(theta) = N(0, I / init_theta_precision)


@dataclass
class linear_gaussian_ssm_wishart_precision:
    """LGSSM observed with an unknown precision MATRIX per series
    (/root/reference/docs/src/manuals/model-specification.md:265-271):
    ``w ~ w_prior; x[1] ~ x0; x[t] ~ N(A x[t-1] + u, P); y[t] ~ N(B x[t], precision = w)``, run with
    ``constraints = q(x, w) = q(x)q(w)``, ``initialization = q(w) = w_init`` and ``iterations``.  ``w_prior`` and
    ``w_init`` are ``Wishart(df, scale)`` as the model writes them; ``x0 = (mean, cov)``."""
    A: np.ndarray
    B: np.ndarray
    P: np.ndarray
    x0: tuple
    w_prior: Wishart
    w_init: Wishart
    u: object = None
    prior_on_previous_state: bool = False


@dataclass
class linear_gaussian_ssm_wishart_noise:
    """LGSSM with an unknown process precision matrix per series, alone or together with an unknown observation precision:
    ``w_p ~ p_prior; w_q ~ q_prior; x[1] ~ x0; x[t] ~ N(A x[t-1] + u, precision = w_p); y[t] ~ N(B x[t], precision = w_q)``,
    run with ``constraints = q(x, w_p, w_q) = q(x)q(w_p)q(w_q)``, ``initialization = q(w_p) = p_init, q(w_q) = q_init`` and
    ``iterations``.  Each noise is either known (``P`` / ``Q``, a covariance) or learned (``*_prior`` and ``*_init`` as
    ``Wishart(df, scale)``, both required); at least one is learned.  ``x0 = (mean, cov)``."""
    A: np.ndarray
    B: np.ndarray
    x0: tuple
    P: np.ndarray = None
    Q: np.ndarray = None
    p_prior: Wishart = None
    p_init: Wishart = None
    q_prior: Wishart = None
    q_init: Wishart = None
    u: object = None
    prior_on_previous_state: bool = False


@dataclass
class linear_gaussian_ssm_continuous_transition:
    """LGSSM that learns its transition matrix per series (RxInfer's ``ContinuousTransition`` with
    ``CTMeta(a -> reshape(a, d, d))``): ``a ~ MvNormal(mean = ma0, covariance = Va0); x[1] ~ x0;
    x[t] ~ ContinuousTransition(x[t-1], a, w_p) (+ u); y[t] ~ N(B x[t], precision = w_q)``, run with
    ``constraints = q(x, a, w_p, w_q) = q(x)q(a)q(w_p)q(w_q)``, ``initialization = q(a) = a_init, ...`` and ``iterations``.
    ``a_prior`` / ``a_init`` are ``(mean, covariance)`` of vec(A) in Julia's column-major order (vec(A)[j d + i] =
    A[i, j]); ``a_init`` is required.  Each noise is known (``P`` / ``Q``, a covariance) or learned (``*_prior`` and
    ``*_init`` as ``Wishart(df, scale)``); both may be known.  ``x0 = (mean, cov)``."""
    B: np.ndarray
    x0: tuple
    a_prior: tuple
    a_init: tuple = None
    P: np.ndarray = None
    Q: np.ndarray = None
    p_prior: Wishart = None
    p_init: Wishart = None
    q_prior: Wishart = None
    q_init: Wishart = None
    u: object = None
    prior_on_previous_state: bool = False


@dataclass
class gaussian_mixture:
    """Gaussian mixture model (RxInfer test/models/mixtures/gmm_multivariate_tests.jl:4-24):
    ``s ~ alpha0; m[k] ~ m_prior[k]; w[k] ~ w_prior[k]; z[i] ~ Categorical(s); y[i] ~ NormalMixture(switch = z[i], m = m,
    p = w)``, run with ``constraints = MeanField()``, ``initialization = {"s": ..., "m": [...], "w": [...]}`` and
    ``iterations``.  Multivariate spelling: ``Dirichlet``, ``MvNormalMeanCovariance``, ``Wishart(df, scale)``.  Univariate
    spelling (gmm_univariate_tests.jl:6-26, K = 2): ``Beta(a, b)`` (= Dirichlet([a, b])), ``NormalMeanVariance``,
    ``GammaShapeRate(shape, rate)`` (= Wishart(2 shape, 1 / (2 rate))), ``vague(Beta)`` / ``vague(GammaShapeRate)``."""
    K: int
    alpha0: object
    m_prior: list
    w_prior: list


class _Marker:
    """An argument that stands for a choice, not a value: every instance of a marker class is equal to every other."""

    def __eq__(self, other):
        return isinstance(other, type(self))

    def __hash__(self):
        return hash(type(self))

    def __repr__(self):
        return f"{type(self).__name__}()"


class MeanField(_Marker):
    """``constraints = MeanField()``: the naive mean-field factorisation q(s) prod q(m[k]) prod q(w[k]) prod q(z[i])."""


class BetheFactorization(_Marker):
    """``BetheFactorization()``: the reference's default constraints (no factorisation of the local joints)."""


def _weights(x, K, what):
    if isinstance(x, Beta):
        if K != 2:
            raise ValueError(f"{what}: Beta weights describe K = 2 components, the model has K = {K}")
        return np.array([float(x.a), float(x.b)])
    if isinstance(x, Dirichlet):
        a = np.asarray(x.alpha, np.float64).reshape(-1)
        if a.shape != (K,):
            raise ValueError(f"{what}: Dirichlet over {a.shape[0]} components, the model has K = {K}")
        return a
    raise TypeError(f"{what}: expected Dirichlet or Beta, got {type(x).__name__}")


def _gaussians(xs, K, what):
    if len(xs) != K:
        raise ValueError(f"{what}: {len(xs)} marginals for K = {K} components")
    mu, V = [], []
    for x in xs:
        if isinstance(x, NormalMeanVariance):
            mu.append(np.array([float(x.m)])); V.append(np.array([[float(x.v)]]))
        elif isinstance(x, MvNormalMeanCovariance):
            mu.append(np.asarray(x.mu, np.float64).reshape(-1)); V.append(np.asarray(x.Sigma, np.float64))
        else:
            raise TypeError(f"{what}: expected NormalMeanVariance or MvNormalMeanCovariance, got {type(x).__name__}")
    return np.stack(mu), np.stack(V)


def _precisions(xs, K, what):
    if len(xs) != K:
        raise ValueError(f"{what}: {len(xs)} marginals for K = {K} components")
    nu, S = [], []
    for x in xs:
        if isinstance(x, GammaShapeRate):          # Gamma(shape a, rate b) = Wishart(2a, 1 / (2b)) in one dimension
            nu.append(2.0 * float(x.a)); S.append(np.array([[1.0 / (2.0 * float(x.b))]]))
        elif isinstance(x, Wishart):
            nu.append(float(x.df)); S.append(np.asarray(x.scale, np.float64))
        else:
            raise TypeError(f"{what}: expected Wishart or GammaShapeRate, got {type(x).__name__}")
    return np.array(nu), np.stack(S)


def _emission_arrays(model, init, K):
    """The NormalMixture emission arrays of the C entries: mu0[K, d], V0[K, d, d] (covariance), nu0[K], S0[K, d, d]
    (Wishart scale) from ``model.m_prior`` / ``model.w_prior``, and the same for the initial q(m), q(w) of ``init``."""
    out = {}
    out["mu0"], out["V0"] = _gaussians(model.m_prior, K, "m_prior")
    out["m_init"], out["Vm_init"] = _gaussians(init["m"], K, "initialization['m']")
    out["nu0"], out["S0"] = _precisions(model.w_prior, K, "w_prior")
    out["nu_init"], out["S_init"] = _precisions(init["w"], K, "initialization['w']")
    d = out["mu0"].shape[1]
    for k in ("m_init", "V0", "Vm_init", "S0", "S_init"):
        if out[k].shape[1] != d:
            raise ValueError(f"{k}: dimension {out[k].shape[1]}, the means have d = {d}")
    return out


def _component_posteriors(r, each, univariate):
    """q(m[k]) and q(w[k]) of every NormalMixture component from a result of the C entry: the last iteration's, or
    with a leading iteration axis (``hist_*``) for ``m`` / ``w`` in ``each``; Normal / Gamma when the model was
    ``univariate``."""
    mp = "hist_" if "m" in each else ""
    wp = "hist_" if "w" in each else ""
    mm, mc, df, iS = r[mp + "m_mean"], r[mp + "m_cov"], r[wp + "w_df"], r[wp + "w_inv_scale"]
    K = mm.shape[-3]
    if univariate:
        return ([NormalMeanVariance(mm[..., k, 0, :], mc[..., k, 0, 0, :]) for k in range(K)],
                [GammaShapeRate(df[..., k, :] / 2, iS[..., k, 0, 0, :] / 2) for k in range(K)])
    return ([MvNormalMeanCovariance(mm[..., k, :, :], mc[..., k, :, :, :]) for k in range(K)],
            [WishartFast(df[..., k, :], iS[..., k, :, :, :]) for k in range(K)])


def gaussian_mixture_arrays(model, initialization):
    """The model and its ``initialization`` in the Dirichlet / MvNormal / Wishart form of the C entry: a dict of host
    arrays alpha0[K], mu0[K, d], V0[K, d, d], nu0[K], S0[K, d, d] and the same for the initial marginals (``*_init``,
    ``Vm_init``), plus ``univariate`` (the model was written with Beta / Normal / Gamma)."""
    K = int(model.K)
    if not isinstance(initialization, dict) or not {"s", "m", "w"} <= set(initialization):
        raise ValueError("gaussian_mixture needs initialization = {'s': q(s), 'm': [q(m[k])], 'w': [q(w[k])]}")
    out = dict(alpha0=_weights(model.alpha0, K, "alpha0"), alpha_init=_weights(initialization["s"], K, "initialization['s']"))
    out.update(_emission_arrays(model, initialization, K))
    out["univariate"] = isinstance(model.alpha0, Beta)
    return out


def check_mean_field(constraints):
    """The mixture node's rules exist for the naive mean-field only, as in the reference (the same message)."""
    if not isinstance(constraints, MeanField):
        raise ValueError("NormalMixture: the factorisation around the node must be the naive mean-field "
                         "q(z) q(s) q(m[1]) ... q(m[K]) q(w[1]) ... q(w[K]); pass constraints = MeanField()")


@dataclass
class hidden_markov_model:
    """Hidden Markov model (RxInfer test/models/statespace/hmm_tests.jl:8-20): ``s_0 ~ Categorical(p0)``,
    ``s[t] ~ DiscreteTransition(s[t-1], A)``, ``x[t] ~ DiscreteTransition(s[t], B)``.  ``A`` (K x K) and ``B`` (M x K) are
    each a ``DirichletCollection`` prior (learned) or a ``PointMass`` probability matrix (known); column j is the
    distribution conditioned on state j.  Run with ``constraints = HMMConstraints()``, ``initialization = {"A": q(A),
    "B": q(B)}`` (``DirichletCollection``, for the learned ones; an ``"s"`` entry is accepted and not needed: every
    iteration starts with the chain) and ``data = {"x": ...}``."""
    p0: object
    A: object
    B: object


class HMMConstraints(_Marker):
    """``q(s, s_0, A, B) = q(s, s_0) q(A) q(B)`` (hmm_tests.jl:22-24): the chain is kept structured, the matrices apart."""


def check_hmm_constraints(constraints):
    if not isinstance(constraints, HMMConstraints):
        raise ValueError("hidden_markov_model runs the structured factorisation q(s, s_0) q(A) q(B) only; pass "
                         f"constraints = HMMConstraints() (got {constraints!r})")


def hmm_symbols(x, M):
    """The observations as symbols: a uint8 index tensor [T, batch] (255 = missing) as it is, or a one-hot float tensor
    [T, M, batch] as the reference passes it (a NaN row is missing).  Soft observations are refused."""
    if x.dtype == torch.uint8:
        if x.dim() != 2:
            raise ValueError(f"data['x'] as symbols must be [T, batch], got {tuple(x.shape)}")
        return x
    if x.dim() != 3 or x.shape[1] != M:
        raise ValueError(f"data['x'] as one-hot vectors must be [T, M = {M}, batch], got {tuple(x.shape)}")
    miss = torch.isnan(x).any(dim=1)
    xx = torch.where(torch.isnan(x), torch.zeros_like(x), x)
    one_hot = ((xx == 0) | (xx == 1)).all(dim=1) & (xx.sum(dim=1) == 1)
    if not bool((one_hot | miss).all()):
        raise ValueError("data['x'] must hold one-hot rows (or NaN for a missing step): soft observations are outside the "
                         "batched hot path")
    sym = xx.argmax(dim=1).to(torch.uint8)
    sym[miss] = 255
    return sym.contiguous()


def _p0(model):
    return np.asarray(model.p0.p if isinstance(model.p0, Categorical) else model.p0, np.float64).reshape(-1)


def _matrix_arguments(model, name, init, K):
    """``{name}_known`` of a ``PointMass`` probability matrix, or ``{name}_prior`` and ``{name}_init`` of a learned
    ``DirichletCollection`` (its q from ``init``); the matrix is K x K for A and M x K for B."""
    v = getattr(model, name)
    if isinstance(v, PointMass):
        out = {f"{name}_known": np.asarray(v.value, np.float64)}
    elif isinstance(v, DirichletCollection):
        if not isinstance(init.get(name), DirichletCollection):
            raise ValueError(f"{name} is learned: pass initialization = {{'{name}': DirichletCollection(...)}}, e.g. "
                             f"vague(DirichletCollection, {np.asarray(v.alpha).shape})")
        out = {f"{name}_prior": np.asarray(v.alpha, np.float64),
               f"{name}_init": np.asarray(init[name].alpha, np.float64)}
        if out[f"{name}_init"].shape != out[f"{name}_prior"].shape:
            raise ValueError(f"initialization['{name}'] has shape {out[f'{name}_init'].shape}, the prior "
                             f"{out[f'{name}_prior'].shape}")
    else:
        raise TypeError(f"model.{name}: expected DirichletCollection or PointMass, got {type(v).__name__}")
    shape = next(iter(out.values())).shape
    if len(shape) != 2 or shape[1] != K or (name == "A" and shape[0] != K):
        raise ValueError(f"model.{name} has shape {shape}; with K = {K} states A is K x K and B is M x K")
    return out


def hmm_arguments(model, initialization):
    """The keyword arguments of ``Context.hmm_vmp`` for ``model`` and ``initialization``."""
    p0 = _p0(model)
    init = initialization or {}
    K = p0.shape[0]
    return {"p0": p0, **_matrix_arguments(model, "A", init, K), **_matrix_arguments(model, "B", init, K)}


@dataclass
class gaussian_hidden_markov_model:
    """Hidden Markov model with Gaussian emissions: ``A ~ DirichletCollection(A_prior)`` (or a ``PointMass`` probability
    matrix, known), ``m[k] ~ m_prior[k]``, ``w[k] ~ w_prior[k]`` (precision), ``s_0 ~ Categorical(p0)``,
    ``s[t] ~ DiscreteTransition(s[t-1], A)``, ``y[t] ~ NormalMixture(switch = s[t], m = m, p = w)``; column j of A is
    p(s_t | s_{t-1} = j), as in ``hidden_markov_model``.  Multivariate spelling: ``MvNormalMeanCovariance`` means and
    ``Wishart(df, scale)`` precisions; at d = 1 also ``NormalMeanVariance`` and ``GammaShapeRate(shape, rate)``
    (= Wishart(2 shape, 1 / (2 rate))).  Run with ``constraints = GaussianHMMConstraints()``, ``initialization =
    {"A": q(A) (A learned), "m": [q(m[k])], "w": [q(w[k])]}`` (an ``"s"`` entry is accepted and not needed) and
    ``data = {"y": [T, d, batch]}`` ([T, batch] at d = 1; an all-NaN step is missing)."""
    p0: object
    A: object
    m_prior: list
    w_prior: list


class GaussianHMMConstraints(_Marker):
    """``q(s_0, s, A, m, w) = q(s_0, s) q(A) q(m[1]) ... q(m[K]) q(w[1]) ... q(w[K])``: the chain kept structured, the
    transition matrix and every state's mean and precision apart."""


def gaussian_hmm_arguments(model, initialization):
    """The keyword arguments of ``Context.hmm_gauss_vmp`` for ``model`` and ``initialization``: p0[K], the A arguments of
    ``hmm_arguments`` and the emission arrays of ``gaussian_mixture_arrays`` (mu0[K, d], V0[K, d, d], nu0[K], S0[K, d, d]
    and the same for the initial q(m), q(w))."""
    p0 = _p0(model)
    init = initialization or {}
    if not {"m", "w"} <= set(init):
        raise ValueError("gaussian_hidden_markov_model needs initialization = {'m': [q(m[k])], 'w': [q(w[k])]} (and 'A' "
                         "when A is learned)")
    return {"p0": p0, **_matrix_arguments(model, "A", init, p0.shape[0]), **_emission_arrays(model, init, p0.shape[0])}


@dataclass
class hgf_offline:
    """``@model hgf_1`` (/root/reference/test/inference/inference_tests.jl:609-622) with every hyper-parameter a number:
    ``ω ~ N(ω_prior)``, ``κ ~ N(κ_prior)``, ``x_0 ~ N(x0_prior)``, ``z[1] ~ N(z1_prior)`` ((mean, variance) each),
    ``z[t] ~ NormalMeanPrecision(z[t-1], z_precision)``, ``x[t] ~ GCV(x[t-1], z[t], κ, ω)`` (variance exp(κ z + ω)),
    ``y[t] ~ NormalMeanVariance(x[t], y_variance)``.  κ and ω are learned per series.  Run with ``constraints =
    MeanField()``, ``initialization = {"κ": ..., "ω": ..., "z": ..., "x": ...}`` (``NormalMeanVariance`` of scalars, as at
    :624-629) and ``data = {"y": [T, batch]}`` (NaN = missing)."""
    κ_prior: tuple = (1.0, 1.0)
    ω_prior: tuple = (0.0, 1.0)
    x0_prior: tuple = (0.0, 1.0)
    z1_prior: tuple = (0.0, 1.0)
    z_precision: float = 1.0
    y_variance: float = 1.0


def hgf_offline_arguments(model, initialization):
    """The ``prior`` and ``init`` arrays of ``Context.hgf_vmp_learn`` for ``model`` and ``initialization``."""
    init = initialization or {}
    missing = [k for k in ("κ", "ω", "z", "x") if not isinstance(init.get(k), NormalMeanVariance)]
    if missing:
        raise ValueError(f"hgf_offline needs initialization = {{'κ', 'ω', 'z', 'x'}} as NormalMeanVariance; missing or not "
                         f"Normal: {missing}")
    scalar = lambda d: (float(np.asarray(d.m)), float(np.asarray(d.v)))
    prior = [float(v) for p in (model.κ_prior, model.ω_prior, model.x0_prior, model.z1_prior) for v in p]
    return dict(prior=prior, init=[v for k in ("κ", "ω", "z", "x") for v in scalar(init[k])],
                z_precision=float(model.z_precision), y_variance=float(model.y_variance))


def vec_order(d):
    """perm with row_major = col_major[perm] (and col_major = row_major[perm]: a transpose is an involution) for vec(A)
    of a d x d matrix: Julia's vec is column-major, the C ABI's a[i * d + j] = A[i, j] row-major."""
    return np.array([(r % d) * d + r // d for r in range(d * d)])


class KeepLast(_Marker):
    """``predictvars`` / ``returnvars`` marker: keep the result of the last iteration (the reference's ``KeepLast()``)."""


class KeepEach(_Marker):
    """``KeepEach()``: keep the result of every iteration.  Predictions per iteration are outside the batched hot path."""


@dataclass
class InferenceResult:
    """``InferenceResult`` (/root/reference/src/inference/batch.jl:18-24)."""
    posteriors: dict
    free_energy: object = None
    model: object = None
    error: object = None
    history: dict = field(default_factory=dict)
    predictions: dict = field(default_factory=dict)
    status: object = None       # per-chain RXG_* codes of a family that returns flagged chains instead of raising


_UNSUPPORTED = ("constraints", "meta", "callbacks", "annotations", "events", "uselock",
                "postprocess", "trace", "benchmark", "free_energy_diagnostics")
_ctx_cache: dict = {}


def default_context(device=None) -> Context:
    dev = torch.cuda.current_device() if device is None else device
    if dev not in _ctx_cache:
        _ctx_cache[dev] = Context(dev)
    ctx = _ctx_cache[dev]
    ctx.bind_stream()
    return ctx


def _predict_keys(predictvars, model, data):
    """Which predictive distributions to return: ``predictvars`` normalised as the reference does
    (src/inference/batch.jl:203-246) -- a bare ``KeepLast()`` stands for every data variable, and a ``y`` with missing
    entries is always predicted.  Only ``KeepLast`` predictions of the LGSSM smoother's ``y`` (observations) and ``o``
    (the ``horizon`` forecasts) run on the batched path; every other form raises ``NotImplementedError``."""
    if isinstance(predictvars, (KeepLast, KeepEach)) and data is None:
        raise ValueError(f"`predictvar` is specified as `{predictvars!r}`, but `data` is not provided. Make sure to provide "
                         "`data` or specify `predictvars` explicitly.")       # the reference's error (batch.jl:210-213)
    if not isinstance(model, linear_gaussian_ssm_smoothing) or isinstance(model, linear_gaussian_ssm_filtering):
        raise NotImplementedError("predictvars: only the smoothing LGSSM predicts on the batched hot path; "
                                  "run this call through stock ReactiveMP")
    if data is None:
        raise NotImplementedError("predictvars / horizon: predictions of the streaming engine (datastream) are outside the "
                                  "batched hot path; pass `data`")
    if isinstance(predictvars, KeepLast):
        predictvars = {k: KeepLast() for k in data if k not in ("ymask", "u")}     # known inputs are not predicted
    if not isinstance(predictvars, dict):
        raise NotImplementedError(f"predictvars={predictvars!r}: expected KeepLast() or a dict of KeepLast() values; "
                                  "run this call through stock ReactiveMP")
    for k, v in predictvars.items():
        if k == "u":
            raise NotImplementedError("predictvars: 'u' holds known inputs, which have no predictive distribution on the "
                                      "batched path")
        if k not in ("y", "o"):
            raise NotImplementedError(f"predictvars: {k!r} is not a data variable of the LGSSM (y, o)")
        if not isinstance(v, KeepLast):
            raise NotImplementedError(f"predictvars[{k!r}] = {v!r}: only KeepLast() predictions run on the batched path")
    if "o" in predictvars and model.horizon <= 0:
        raise ValueError("predictvars: 'o' (the forecasts) needs linear_gaussian_ssm_smoothing(..., horizon > 0)")
    keys = set(predictvars)
    mask = data.get("ymask")
    if mask is not None and not bool((torch.as_tensor(mask) != 0).all()):
        keys.add("y")                                  # data with missing entries are predicted (batch.jl:231-245)
    return keys


# --------------------------------------------------------------------------- Delta node (nonlinear maps)
@dataclass
class CudaFunction:
    """A user function for a Delta node: CUDA C++ ``source`` defining
    ``template <class S> __device__ void <name>(const S* x, S* z)`` from R^d_in to R^d_out, with math functions called
    unqualified (the library instantiates it with dual numbers for Linearization and with double for Unscented)."""
    source: str
    name: str
    d_in: int
    d_out: int


class Linearization(_Marker):
    """``Linearization()``: the Delta node's messages from the first-order Taylor expansion at the incoming mean
    (Jacobians by forward-mode dual numbers, fp32)."""


@dataclass(frozen=True)
class Unscented:
    """``Unscented(alpha=, beta=, kappa=)``: the unscented transform with 2d + 1 sigma points (fp64); the defaults are
    ReactiveMP's."""
    alpha: float = 1e-3
    beta: float = 2.0
    kappa: float = 0.0


@dataclass
class nonlinear_gaussian_ssm_smoothing:
    """``x[1] ~ x0; x[t] ~ N(f(x[t-1]), P); y[t] ~ N(B x[t], Q)`` or ``N(g(x[t]), Q)``, the Delta node ``f`` (and ``g``)
    approximated as ``meta`` says [ref: test/models/nonlinear/].  ``x0 = (mean, cov)``."""
    f: CudaFunction
    P: np.ndarray
    Q: np.ndarray
    x0: tuple
    B: np.ndarray = None
    g: CudaFunction = None


@dataclass
class nonlinear_gaussian_ssm_filtering(nonlinear_gaussian_ssm_smoothing):
    """The one-step model with ``@autoupdates`` of ``mean_cov(q(x_t))``: every datum pushes the carry through f (and
    P) before its observation; ``x0`` initialises the carry."""


@dataclass
class nonlinear_gamma_streaming:
    """The paper's pendulum (paper/example.jl): ``previous_state ~ MvNormal(prior)``, ``state ~ f(previous_state)``,
    ``noise ~ Gamma(shape, scale)``, ``observation ~ Normal(dot(c, state), precision = noise)`` with
    ``q(state, noise) = q(state) q(noise)`` and the priors autoupdated from q(state) and q(noise).  ``state0 = (mean,
    cov)`` and ``noise0 = (shape, scale)`` are the initial marginals (and the first datum's priors); ``P`` an optional
    process noise added to the Delta node's message (the paper has none)."""
    f: CudaFunction
    c: np.ndarray
    state0: tuple = ((0.5, 0.0), ((0.01, 0.0), (0.0, 0.01)))
    noise0: tuple = (1.0, 100.0)
    P: np.ndarray = None


_DELTA_MODELS = (nonlinear_gaussian_ssm_smoothing, nonlinear_gamma_streaming)


def delta_method(model, meta):
    """The one approximation ``meta`` assigns to the model's Delta nodes: (method code, (alpha, beta, kappa) or None)."""
    if not isinstance(meta, dict):
        raise ValueError("meta: expected a dict {'f': Linearization() or Unscented(...), 'g': ...}")
    nodes = ["f"] + (["g"] if getattr(model, "g", None) is not None else [])
    bad = set(meta) - set(nodes)
    if bad:
        raise ValueError(f"meta: {sorted(bad)} are not Delta nodes of {type(model).__name__} (its nodes: {nodes})")
    methods = []
    for n in nodes:
        m = meta.get(n)
        if not isinstance(m, (Linearization, Unscented)):
            # the reference refuses a Delta node without an approximation method between Gaussian nodes
            raise ValueError(f"meta: the Delta node {n!r} needs an approximation method: Linearization() or Unscented()")
        methods.append(m)
    if any(m != methods[0] for m in methods[1:]):
        raise NotImplementedError("meta: f and g with different approximation methods are outside the batched hot path")
    m = methods[0]
    if isinstance(m, Linearization):
        return L.RXG_DELTA_LINEARIZATION, None
    return L.RXG_DELTA_UNSCENTED, (float(m.alpha), float(m.beta), float(m.kappa))


def delta_module(ctx, model, meta):
    """The compiled module of the model's Delta nodes (cached by the context)."""
    method, ut = delta_method(model, meta)
    f, g = model.f, getattr(model, "g", None)
    d = f.d_in
    if f.d_out != d:
        raise ValueError(f"f maps R^{f.d_in} to R^{f.d_out}: a transition maps R^d to R^d")
    m = 1
    if g is not None:
        if g.d_in != d:
            raise ValueError(f"g takes R^{g.d_in}, the state is R^{d}")
        m = g.d_out
    elif getattr(model, "B", None) is not None:
        m = np.atleast_2d(np.asarray(model.B)).shape[0]
    elif not isinstance(model, nonlinear_gamma_streaming):
        raise ValueError("the observation needs B (linear) or g (a CudaFunction)")
    source = f.source if g is None or g.source == f.source else f.source + "\n" + g.source
    return ctx.delta_model(source, f.name, d, m, method, g_name=None if g is None else g.name, ut=ut)


def _check_delta_constraints(constraints):
    if not isinstance(constraints, MeanField):
        raise NotImplementedError("nonlinear_gamma_streaming runs under q(state, noise) = q(state) q(noise): pass "
                                  "constraints = MeanField()")


def _infer_delta(model, *, data, meta, initialization, free_energy, iterations, returnvars, predictvars, datastream,
                 autoupdates, keephistory, historyvars, autostart, batch, context, **_):
    if initialization is not None:
        where = "state0 = (mean, cov) and noise0 = (shape, scale)" if isinstance(model, nonlinear_gamma_streaming) \
            else "x0 = (mean, cov)"
        raise NotImplementedError(f"initialization: {type(model).__name__} takes its initial marginals as model fields "
                                  f"({where})")
    if returnvars is not None and not isinstance(returnvars, KeepLast):
        raise NotImplementedError("returnvars: the nonlinear state-space models return the last marginals (KeepLast()); "
                                  "per-iteration results are outside the batched hot path")
    if free_energy:
        raise NotImplementedError("free_energy: the Delta node's energy term under Linearization / Unscented is not "
                                  "restated on the batched path")
    if predictvars is not None:
        raise NotImplementedError("predictvars: predictions of the nonlinear state-space models are outside the "
                                  "batched hot path")
    if meta is None:
        raise ValueError("meta: the Delta nodes need an approximation method, e.g. meta = {'f': Linearization()}")
    delta_method(model, meta)           # refuse a bad meta before anything runs
    smoothing = type(model) is nonlinear_gaussian_ssm_smoothing
    if smoothing and iterations not in (None, 1):
        raise NotImplementedError("iterations > 1 on the tree-structured smoother repeats the same schedule")
    if data is None:
        if smoothing:
            raise ValueError("nonlinear_gaussian_ssm_smoothing runs over whole series: pass data = {'y': [T, m, batch]}")
        if datastream is None and autoupdates is None:
            raise ValueError("either `data` or `datastream` (or `autoupdates` for a push-driven engine) is required")
        if batch is None:
            raise ValueError("streaming inference needs `batch` (number of lock-step datastreams)")
        from .streaming import RxInferenceEngine
        return RxInferenceEngine(context or default_context(), model, batch=batch, iterations=iterations,
                                 keephistory=keephistory, historyvars=historyvars, datastream=datastream,
                                 autostart=autostart, meta=meta)
    if "y" not in data:
        raise KeyError("data must contain the observations under key 'y'")

    def run(ctx):
        y = torch.as_tensor(data["y"], device=f"cuda:{ctx.device}", dtype=torch.float32).contiguous()
        mask = data.get("ymask")
        mod = delta_module(ctx, model, meta)
        if smoothing:
            r = ctx.delta_smooth(mod, y, model.x0[0], model.x0[1], model.P, model.Q, B=model.B, mask=mask)
            _raise_flagged(r["status"], "nonlinear_gaussian_ssm_smoothing: ",
                           " (NOT_SPD: a predicted or innovation covariance is not SPD; NAN: a non-finite value)")
            return InferenceResult(posteriors={"x": MvNormalMeanCovariance(r["mean"], r["cov"])}, model=model)
        from .streaming import RxInferenceEngine
        eng = RxInferenceEngine(ctx, model, batch=y.shape[-1], iterations=iterations, keephistory=y.shape[0],
                                historyvars=historyvars, datastream=None, autostart=False, meta=meta)
        eng.push(y if mask is None else {"y": y, "ymask": mask})
        return InferenceResult(posteriors={}, history=eng.history, model=model)
    return run


def _raise_flagged(status, prefix="", suffix=""):
    """Raise ``RxGaussError`` when the kernel flagged some chains: RXG_ERR_NOT_SPD if any chain is NOT_SPD, else the first
    flagged chain's code; the message counts the chains and names the codes."""
    bad = status != 0
    if bool(bad.any()):
        codes = sorted({L.STATUS_NAMES.get(int(c), str(int(c))) for c in status[bad].unique().tolist()})
        raise L.RxGaussError(L.RXG_ERR_NOT_SPD if "NOT_SPD" in codes else int(status[bad][0]),
                             f"{prefix}{int(bad.sum())} of {bad.numel()} chains flagged {codes}{suffix}")


def _noise_kwargs(model):
    """The P / Q arguments of ``Context.lgssm_vmp_noise`` / ``lgssm_vmp_transition`` from a model whose noises are each
    known (``P`` / ``Q``) or learned (``*_prior`` / ``*_init`` as ``Wishart``)."""
    kw = {}
    for name in ("p", "q"):
        known, prior, init = getattr(model, name.upper()), getattr(model, f"{name}_prior"), getattr(model, f"{name}_init")
        if known is not None and (prior is not None or init is not None):
            raise ValueError(f"{name.upper()} is known: pass either {name.upper()} or {name}_prior / {name}_init")
        if known is not None:
            kw[name.upper()] = known
        elif prior is not None and init is not None:
            kw[f"{name}_prior"], kw[f"{name}_init"] = (prior.df, prior.inv_scale()), init.mean()
        else:
            kw[f"{name}_prior"], kw[f"{name}_init"] = prior, init    # Context names what is missing
    return kw


def _noise_posteriors(r):
    """``w_p`` / ``w_q`` of the learned precisions from a noise-learning result (KeepEach: leading iteration axis)."""
    return {f"w_{name}": WishartFast(r[f"df_{name}"], r[f"inv_scale_{name}"]) for name in ("p", "q")
            if r[f"df_{name}"] is not None}


def _kept_each(who, returnvars, names, each=None, bare_each=True, by_name=True):
    """The variables of ``names`` that ``returnvars`` keeps for every iteration.  ``returnvars`` is None or KeepLast()
    (every variable, last iteration only), KeepEach() (every variable of ``each``, by default all of ``names``; refused
    unless ``bare_each``) or, with ``by_name``, a dict of KeepLast() / KeepEach() by variable, KeepEach() only for
    ``each``.  Every other form raises ``NotImplementedError``."""
    each = set(names if each is None else each)
    if isinstance(returnvars, dict) and by_name:
        if set(returnvars) - set(names) or not all(isinstance(v, (KeepEach, KeepLast)) for v in returnvars.values()):
            raise NotImplementedError(f"returnvars={returnvars!r}: KeepLast() of {', '.join(names)}; KeepEach() of "
                                      f"{', '.join(n for n in names if n in each)}")
        kept = {k for k, v in returnvars.items() if isinstance(v, KeepEach)}
        if kept - each:
            last = sorted(kept - each)
            raise NotImplementedError(f"returnvars: {', '.join(f'q({k})' for k in last)} kept for the last iteration "
                                      "only (KeepLast)")
        return kept
    if returnvars is None or isinstance(returnvars, KeepLast):
        return set()
    if bare_each and isinstance(returnvars, KeepEach):
        return each
    forms = ["KeepLast()"] + ["KeepEach()"] * bare_each + [f"a dict over {', '.join(names)}"] * by_name
    raise NotImplementedError(f"returnvars={returnvars!r}: {who} returns {' or '.join(forms)}")


# --------------------------------------------------------------------------- handlers of infer()
# Every handler takes the model and the keywords of ``infer`` (each keeps the ones it uses) and runs the refusals of its
# model; they raise.  It returns a streaming engine, or ``run(ctx)``, the device work, which ``infer`` runs under the
# ``catch_exception`` guard.
def _infer_hmm(model, *, data, initialization, iterations, free_energy, returnvars, **_):
    """``infer`` of ``hidden_markov_model``: one ``rxg_hmm_vmp_f32`` launch.  ``returnvars`` is KeepLast() / KeepEach() for
    every variable or a dict over ``s``, ``A``, ``B``; ``s_0`` is the last iteration's."""
    if data is None or "x" not in data:
        raise KeyError("hidden_markov_model needs data = {'x': observations}")
    each = _kept_each("hidden_markov_model", returnvars, ("s", "A", "B", "s_0"), each=("s", "A", "B"))
    args = hmm_arguments(model, initialization)
    M = (args["B_known"] if "B_known" in args else args["B_prior"]).shape[0]
    x = hmm_symbols(torch.as_tensor(data["x"]), M)

    def run(ctx):
        r = ctx.hmm_vmp(x.to(f"cuda:{ctx.device}").contiguous(), **args, iterations=iterations or 1,
                        want_free_energy=bool(free_energy), keep_each=bool(each))
        _raise_flagged(r["status"], "hidden_markov_model: ", " (BAD_ARG: a symbol >= M; NAN: data impossible under the model)")
        post = {"s": Categorical(r["hist_s"] if "s" in each else r["s_prob"]), "s_0": Categorical(r["s0_prob"])}
        for name in ("A", "B"):
            if r[f"{name}_alpha"] is not None:
                post[name] = DirichletCollection(r[f"hist_{name}"] if name in each else r[f"{name}_alpha"])
        return InferenceResult(posteriors=post, model=model, free_energy=r["free_energy"])
    return run


def _check_gaussian_hmm_constraints(constraints):
    if not isinstance(constraints, GaussianHMMConstraints):
        raise ValueError("gaussian_hidden_markov_model runs the structured factorisation q(s_0, s) q(A) q(m[1]) ... q(m[K]) "
                         f"q(w[1]) ... q(w[K]) only; pass constraints = GaussianHMMConstraints() (got {constraints!r})")


def _infer_hmm_gauss(model, *, data, initialization, iterations, free_energy, returnvars, **_):
    """``infer`` of ``gaussian_hidden_markov_model``: one ``rxg_hmm_gauss_vmp_f32`` launch.  ``returnvars`` is
    KeepLast() / KeepEach() for every variable or a dict over ``s``, ``A``, ``m``, ``w`` (and KeepLast() of ``s_0``)."""
    if "y" not in data:
        raise KeyError("gaussian_hidden_markov_model needs data = {'y': observations}")
    each = _kept_each("gaussian_hidden_markov_model", returnvars, ("s", "A", "m", "w", "s_0"),
                      each=("s", "A", "m", "w"))
    args = gaussian_hmm_arguments(model, initialization)
    d = args["mu0"].shape[1]
    y = torch.as_tensor(data["y"])
    y = y[:, None] if y.dim() == 2 and d == 1 else y            # univariate data may come as [T, batch]
    if y.dim() != 3 or y.shape[1] != d:
        raise ValueError(f"data['y'] must be [T, d = {d}, batch] (or [T, batch] at d = 1), got {tuple(y.shape)}")
    univariate = isinstance(model.m_prior[0], NormalMeanVariance) and isinstance(model.w_prior[0], GammaShapeRate)

    def run(ctx):
        r = ctx.hmm_gauss_vmp(y.to(device=f"cuda:{ctx.device}", dtype=torch.float32).contiguous(), **args,
                              iterations=iterations or 1, want_free_energy=bool(free_energy), keep_each=bool(each))
        _raise_flagged(r["status"], "gaussian_hidden_markov_model: ",
                       " (BAD_ARG: a non-finite datum other than an all-NaN step; NAN: a vanished normaliser; NOT_SPD: "
                       "an update met a non-SPD matrix)")
        post = {"s": Categorical(r["hist_s"] if "s" in each else r["s_prob"]), "s_0": Categorical(r["s0_prob"])}
        if r["A_alpha"] is not None:
            post["A"] = DirichletCollection(r["hist_A"] if "A" in each else r["A_alpha"])
        post["m"], post["w"] = _component_posteriors(r, each, univariate)
        return InferenceResult(posteriors=post, model=model, free_energy=r["free_energy"])
    return run


@dataclass
class binomial_regression:
    """Bayesian binomial / logistic regression (RxInfer test/models/regression/binomialreg_tests.jl:32-43):
    ``β ~ MvNormalWeightedMeanPrecision(prior_xi, prior_precision)``, ``y[i] ~ BinomialPolya(X[i], n_trials[i], β)``, i.e.
    y_i ~ Binomial(n_i, σ(X_iᵀβ)), fitted by mean-field Pólya-Gamma VMP (DESIGN 3.21).  Run with ``data = {"X": [batch, N,
    p], "y": [batch, N], "n_trials": [batch, N]}`` (no ``n_trials``: every n = 1, logistic regression; one series may
    come without the batch axis); a sample with n = 0 contributes nothing."""
    prior_xi: object
    prior_precision: object


def _infer_binomial(model, *, data, initialization, iterations, free_energy, returnvars, **_):
    """``infer`` of ``binomial_regression``: one ``rxg_binomial_polya_vmp_f32`` launch.  ``returnvars`` is KeepLast() /
    KeepEach() of ``β``; ``free_energy=True`` gives F after every iteration."""
    if initialization is not None:
        raise NotImplementedError("binomial_regression starts from the prior: initialization is not used")
    if "X" not in data or "y" not in data:
        raise KeyError("binomial_regression needs data = {'X': [batch, N, p], 'y': [batch, N]} (and 'n_trials')")
    bad = set(data) - {"X", "y", "n_trials"}
    if bad:
        raise ValueError(f"binomial_regression: unknown data {sorted(bad)} (X, y, n_trials)")
    each = bool(_kept_each("binomial_regression", returnvars, ("β",)))
    X = torch.as_tensor(data["X"])
    single = X.dim() == 2
    X = X[None] if single else X
    if X.dim() != 3:
        raise ValueError(f"data['X'] must be [batch, N, p] (or [N, p]), got {tuple(X.shape)}")
    nb, N, p = X.shape

    def counts(name):
        v = torch.as_tensor(data[name])
        v = v[None] if single else v
        if tuple(v.shape) != (nb, N):
            raise ValueError(f"data['{name}'] must be [batch, N] = {(nb, N)} (or [N]), got {tuple(v.shape)}")
        if v.is_floating_point() and not bool((v == torch.round(v)).all()):
            raise ValueError(f"data['{name}'] must hold whole numbers")
        return v.to(torch.int32)

    y = counts("y")
    n = counts("n_trials") if data.get("n_trials") is not None else None

    def run(ctx):
        dev = f"cuda:{ctx.device}"
        r = ctx.binomial_polya_vmp(X.to(device=dev, dtype=torch.float32).permute(1, 2, 0).contiguous(),
                                   y.to(dev).T.contiguous(), model.prior_xi, model.prior_precision,
                                   ntrials=None if n is None else n.to(dev).T.contiguous(), iterations=iterations or 1,
                                   want_free_energy=bool(free_energy), keep_each=each)
        _raise_flagged(r["status"], "binomial_regression: ", " (BAD_ARG: a non-finite x, y < 0, n < 0 or y > n; NOT_SPD: "
                       "a non-positive pivot; NAN: a non-finite result)")
        mean, cov = (r["hist_mean"], r["hist_cov"]) if each else (r["beta_mean"], r["beta_cov"])
        fe = r["free_energy"]
        if single:
            mean, cov, fe = mean[..., 0], cov[..., 0], (fe[:, 0] if fe is not None else None)
        return InferenceResult(posteriors={"β": MvNormalMeanCovariance(mean, cov)}, model=model, free_energy=fe)
    return run


@dataclass
class gamma_mixture:
    """Gamma mixture model (RxInfer test/models/mixtures/gamma_mixture_tests.jl:7-40): ``s ~ prior_s``,
    ``as[k] ~ Gamma(shape, rate of priors_as[k])``, ``bs[k] ~ Gamma(shape, rate of priors_bs[k])``, ``z[i] ~
    Categorical(s)``, ``y[i] ~ GammaMixture(switch = z[i], a = as, b = bs)`` (component k: Gamma(shape as[k], rate
    bs[k])), fitted by mean-field VMP with point-mass shapes (DESIGN 3.24).  ``prior_s`` is a ``Dirichlet``, the priors
    ``GammaShapeRate``; every shape prior needs shape >= 1.  Run with ``constraints = GammaMixtureConstraints(a_start)``,
    ``initialization = {"s": Dirichlet, "z": vague(Categorical, K), "bs": GammaShapeRate or a list of K}`` and
    ``data = {"y": [N, batch]}`` (one data set may come as [N])."""
    K: int
    prior_s: object
    priors_as: list
    priors_bs: list


@dataclass(frozen=True)
class GammaMixtureConstraints:
    """``q(z, as, bs, s) = q(z)q(as)q(bs)q(s)`` with every q(as[k]) and q(bs[k]) apart and ``q(as)::
    PointMassFormConstraint(starting_point = a_start)`` (gamma_mixture_tests.jl:35-42): the shapes are MAP points, found
    by Newton's method from ``a_start`` (a number, or one per component)."""
    a_start: object = 1.0


def _check_gamma_mixture_constraints(constraints):
    if not isinstance(constraints, GammaMixtureConstraints):
        raise ValueError("gamma_mixture runs q(z) q(as) q(bs) q(s) with q(as)::PointMassFormConstraint only: the Gamma "
                         "shape has no conjugate posterior, so q(as) must be a point mass; pass constraints = "
                         f"GammaMixtureConstraints(a_start=...) (got {constraints!r})")


def _gamma_params(xs, K, what):
    xs = list(xs) if isinstance(xs, (list, tuple)) else [xs] * K
    if len(xs) != K:
        raise ValueError(f"{what}: {len(xs)} marginals for K = {K} components")
    if not all(isinstance(x, GammaShapeRate) for x in xs):
        raise TypeError(f"{what}: expected GammaShapeRate, got {[type(x).__name__ for x in xs]}")
    return np.array([float(x.a) for x in xs]), np.array([float(x.b) for x in xs])


def gamma_mixture_arguments(model, constraints, initialization):
    """The host arrays [K] of ``Context.gamma_mixture_vmp`` (``Context.GAMMA_MIXTURE_KEYS``) from the model, its
    constraints and ``initialization``; refuses what the batched path does not run."""
    K = int(model.K)
    if not 2 <= K <= 8:
        raise NotImplementedError(f"gamma_mixture: K = {K} components; the batched path runs 2 <= K <= 8")
    if not isinstance(model.prior_s, Dirichlet):
        raise TypeError(f"prior_s: expected Dirichlet, got {type(model.prior_s).__name__}")
    out = dict(alpha_s=_weights(model.prior_s, K, "prior_s"))
    out["a_shape0"], out["a_rate0"] = _gamma_params(model.priors_as, K, "priors_as")
    out["b_shape0"], out["b_rate0"] = _gamma_params(model.priors_bs, K, "priors_bs")
    if (out["a_shape0"] < 1.0).any():
        raise NotImplementedError(f"priors_as: shape {out['a_shape0'].min()} < 1; the batched path needs every shape prior "
                                  ">= 1, where the point-mass objective is concave and its maximiser unique")
    a0 = np.broadcast_to(np.asarray(constraints.a_start, np.float64).reshape(-1), (K,)).copy() \
        if np.size(constraints.a_start) in (1, K) else None
    if a0 is None or not (np.isfinite(a0) & (a0 > 0)).all():
        raise ValueError(f"GammaMixtureConstraints: a_start must be one positive number or {K}, got {constraints.a_start!r}")
    out["a_start"] = a0
    if not isinstance(initialization, dict) or not {"s", "bs"} <= set(initialization):
        raise ValueError("gamma_mixture needs initialization = {'s': Dirichlet, 'z': vague(Categorical, K), 'bs': "
                         "GammaShapeRate or a list}")
    bad = set(initialization) - {"s", "z", "bs"}
    if bad:
        raise ValueError(f"initialization: {sorted(bad)} are not initialised on this model (s, z, bs; as has its "
                         "starting point in the constraints)")
    if not isinstance(initialization["s"], Dirichlet):
        raise TypeError(f"initialization['s']: expected Dirichlet, got {type(initialization['s']).__name__}")
    out["alpha_init"] = _weights(initialization["s"], K, "initialization['s']")
    z = initialization.get("z")
    if z is not None:
        p = np.asarray(z.p if isinstance(z, Categorical) else np.nan, np.float64).reshape(-1)
        if not isinstance(z, Categorical) or p.shape != (K,) or not np.allclose(p, 1.0 / K, rtol=0, atol=1e-12):
            raise NotImplementedError("initialization['z']: the batched path starts from the uniform q(z) = "
                                      f"vague(Categorical, {K})")
    out["b_shape_init"], out["b_rate_init"] = _gamma_params(initialization["bs"], K, "initialization['bs']")
    for k, v in out.items():
        if not (np.isfinite(v) & (v > 0)).all():
            raise ValueError(f"gamma_mixture: {k} must be positive and finite, got {v}")
    return out


def _infer_gamma_mixture(model, *, data, constraints, initialization, iterations, free_energy, returnvars, **_):
    """``infer`` of ``gamma_mixture``: one ``rxg_gamma_mixture_vmp_f32`` launch.  ``returnvars`` is KeepLast() /
    KeepEach() or a dict over ``s``, ``z``, ``as``, ``bs``, KeepEach() for ``as`` and ``bs`` (a leading iteration
    axis)."""
    if "y" not in data:
        raise KeyError("gamma_mixture needs data = {'y': [N, batch]}")
    bad = set(data) - {"y"}
    if bad:
        raise ValueError(f"gamma_mixture: unknown data {sorted(bad)} (y)")
    each = _kept_each("gamma_mixture", returnvars, ("s", "z", "as", "bs"), each=("as", "bs"))
    args = gamma_mixture_arguments(model, constraints, initialization)
    y = torch.as_tensor(data["y"])
    single = y.dim() == 1
    y = y[:, None] if single else y
    if y.dim() != 2:
        raise ValueError(f"data['y'] must be [N, batch] (or [N]), got {tuple(y.shape)}")
    K = int(model.K)

    def run(ctx):
        r = ctx.gamma_mixture_vmp(y.to(device=f"cuda:{ctx.device}", dtype=torch.float32).contiguous(),
                                  *(args[k] for k in Context.GAMMA_MIXTURE_KEYS), iterations=iterations or 1,
                                  want_free_energy=bool(free_energy), want_z=True, keep_each=bool(each))
        _raise_flagged(r["status"], "gamma_mixture: ", " (BAD_ARG: a datum <= 0 or not finite; NAN: a shape's Newton "
                                                       "iteration did not converge)")
        a = r["hist_a"] if "as" in each else r["a_hat"]
        bs, br = (r["hist_b_shape"], r["hist_b_rate"]) if "bs" in each else (r["b_shape"], r["b_rate"])
        sq = (lambda t: t[..., 0]) if single else (lambda t: t)          # one data set: no batch axis
        post = {"s": Dirichlet(sq(r["alpha"])), "z": Categorical(sq(r["z_prob"])),
                "as": [PointMass(sq(a[..., k, :])) for k in range(K)],
                "bs": [GammaShapeRate(sq(bs[..., k, :]), sq(br[..., k, :])) for k in range(K)]}
        fe = r["free_energy"]
        return InferenceResult(posteriors=post, model=model, free_energy=None if fe is None else sq(fe))
    return run


@dataclass
class multinomial_regression:
    """Bayesian multinomial regression (RxInfer test/models/regression/multinomialreg_tests.jl, offline item):
    ``ψ ~ MvNormalWeightedMeanPrecision(prior_xi, prior_precision)``, ``y[i] ~ MultinomialPolya(N_i, ψ)`` with N_i the sum
    of y[i]'s K counts and ψ of length K − 1 (stick-breaking), fitted by mean-field Pólya-Gamma VMP (DESIGN 3.22).  Run
    with ``data = {"y": [batch, n, K]}`` (one data set may come as [n, K]); an all-zero sample contributes nothing."""
    prior_xi: object
    prior_precision: object


@dataclass
class multinomial_regression_online:
    """The same model online (multinomialreg_tests.jl, online item): ``ψ ~ MvNormalWeightedMeanPrecision(ξ_ψ, W_ψ)``,
    ``y ~ MultinomialPolya(N, ψ)`` with ``@autoupdates ξ_ψ, W_ψ = weightedmean_precision(q(ψ))`` and
    ``initialization = {"ψ": MvNormalWeightedMeanPrecision(ξ, W)}``.  ``infer`` returns an ``RxInferenceEngine`` whose
    chunks are int32 counts [Tc, K, batch]; ``data = {"y": [batch, T, K]}`` (or [T, K]) gives a completed engine."""


def _counts(v, what):
    """Whole-number counts as an int32 tensor; a float array must hold whole numbers."""
    v = torch.as_tensor(v)
    if v.is_floating_point():
        if not bool((v == torch.round(v)).all()):
            raise ValueError(f"{what} must hold whole numbers")
    elif v.dtype == torch.bool or v.is_complex():
        raise ValueError(f"{what} must hold whole numbers")
    return v.to(torch.int32)


def _infer_multinomial(model, *, data, initialization, iterations, free_energy, returnvars, **_):
    """``infer`` of ``multinomial_regression``: one ``rxg_multinomial_polya_vmp_f32`` call.  ``returnvars`` is
    KeepLast() / KeepEach() of ``ψ``; ``free_energy=True`` gives F after every iteration."""
    if initialization is not None:
        raise NotImplementedError("multinomial_regression starts from the prior: initialization is not used")
    if "y" not in data:
        raise KeyError("multinomial_regression needs data = {'y': [batch, n, K]}")
    bad = set(data) - {"y"}
    if bad:
        raise ValueError(f"multinomial_regression: unknown data {sorted(bad)} (y)")
    each = bool(_kept_each("multinomial_regression", returnvars, ("ψ",)))
    y = _counts(data["y"], "data['y']")
    single = y.dim() == 2
    y = y[None] if single else y
    if y.dim() != 3:
        raise ValueError(f"data['y'] must be [batch, n, K] (or [n, K]), got {tuple(y.shape)}")

    def run(ctx):
        r = ctx.multinomial_polya_vmp(y.to(f"cuda:{ctx.device}").permute(1, 2, 0).contiguous(), model.prior_xi,
                                      model.prior_precision, iterations=iterations or 1,
                                      want_free_energy=bool(free_energy), keep_each=each)
        _raise_flagged(r["status"], "multinomial_regression: ", " (BAD_ARG: a negative count; NOT_SPD: a non-positive "
                       "pivot; NAN: a non-finite result)")
        mean, cov = (r["hist_mean"], r["hist_cov"]) if each else (r["psi_mean"], r["psi_cov"])
        fe = r["free_energy"]
        if single:
            mean, cov, fe = mean[..., 0], cov[..., 0], (fe[:, 0] if fe is not None else None)
        return InferenceResult(posteriors={"ψ": MvNormalMeanCovariance(mean, cov)}, model=model, free_energy=fe)
    return run


def _infer_multinomial_online(model, *, data, initialization, autoupdates, iterations, free_energy, returnvars,
                              predictvars, keephistory, historyvars, datastream, autostart, batch, context, **_):
    """``infer`` of ``multinomial_regression_online``: an ``RxInferenceEngine`` of kind "multinomial" (the carry q(ψ) in
    fp64 on the device).  With ``data`` the whole stream is one chunk and the engine is returned completed."""
    if predictvars is not None or returnvars is not None:
        raise NotImplementedError("multinomial_regression_online keeps q(ψ) through keephistory; returnvars and "
                                  "predictvars are outside the batched hot path")
    if autoupdates is None:
        raise ValueError("multinomial_regression_online needs autoupdates (ξ_ψ, W_ψ = weightedmean_precision(q(ψ)))")
    init = initialization.get("ψ") if isinstance(initialization, dict) else None
    if not isinstance(init, MvNormalWeightedMeanPrecision) or set(initialization) != {"ψ"}:
        raise ValueError("multinomial_regression_online needs initialization = {'ψ': MvNormalWeightedMeanPrecision(ξ, W)}")
    from .streaming import RxInferenceEngine
    y = None
    if data is not None:
        if set(data) != {"y"}:
            raise ValueError(f"multinomial_regression_online: data must be {{'y': [batch, T, K]}}, got {sorted(data)}")
        y = _counts(data["y"], "data['y']")
        y = y[None] if y.dim() == 2 else y
        if y.dim() != 3:
            raise ValueError(f"data['y'] must be [batch, T, K] (or [T, K]), got {tuple(y.shape)}")
        if batch is not None and batch != y.shape[0]:
            raise ValueError(f"batch = {batch}, data['y'] has {y.shape[0]} series")
    elif batch is None:
        raise ValueError("streaming inference needs `batch` (number of lock-step datastreams)")
    ctx = context or default_context()
    if y is not None:
        datastream, batch, autostart = [y.to(f"cuda:{ctx.device}").permute(1, 2, 0).contiguous()], y.shape[0], True
    return RxInferenceEngine(ctx, model, batch=batch, iterations=iterations, keephistory=keephistory,
                             historyvars=historyvars, free_energy=free_energy, datastream=datastream, autostart=autostart,
                             initialization=init)


def _check_hgf_offline_constraints(constraints):
    if not isinstance(constraints, MeanField):
        raise ValueError(f"hgf_offline runs the naive mean-field factorisation only; pass constraints = MeanField() "
                         f"(got {constraints!r})")


def _infer_hgf_offline(model, *, data, initialization, iterations, free_energy, returnvars, **_):
    """``infer`` of ``hgf_offline``: one ``rxg_hgf_vmp_learn_f32`` launch.  ``returnvars``: KeepLast() for x, z (and x_0),
    KeepEach() or KeepLast() for κ, ω.  A chain whose GH products collapse (DESIGN 3.19) is flagged RXG_ERR_NAN in
    ``result.status[batch]`` and its posteriors are not meaningful; the call does not raise for it, since at large batches
    a few such chains are expected and the others' results stand."""
    if "y" not in data:
        raise KeyError("hgf_offline needs data = {'y': observations}")
    each = _kept_each("hgf_offline", returnvars, ("x", "z", "x_0", "κ", "ω"), each=("κ", "ω"), bare_each=False)
    args = hgf_offline_arguments(model, initialization)

    def run(ctx):
        y = torch.as_tensor(data["y"]).to(device=f"cuda:{ctx.device}", dtype=torch.float32).contiguous()
        if y.dim() != 2:
            raise ValueError(f"data['y'] must be [T, batch], got {tuple(y.shape)}")
        r = ctx.hgf_vmp_learn(y, **args, iterations=iterations or 1, want_free_energy=bool(free_energy),
                              keep_each=bool(each))
        post = {"x": NormalMeanVariance(r["xz"][:, 0], r["xz"][:, 1]), "z": NormalMeanVariance(r["xz"][:, 2], r["xz"][:, 3]),
                "x_0": NormalMeanVariance(r["x0"][0], r["x0"][1])}
        for i, name in enumerate(("κ", "ω")):
            q = r["hist_kw"] if name in each else r["kw"]     # KeepEach: a leading iteration axis
            post[name] = NormalMeanVariance(q[..., i, 0, :], q[..., i, 1, :])
        return InferenceResult(posteriors=post, model=model, free_energy=r["free_energy"], status=r["status"])
    return run


_WISHART_LGSSMS = (linear_gaussian_ssm_wishart_precision, linear_gaussian_ssm_wishart_noise,
                   linear_gaussian_ssm_continuous_transition)


def _series(run):
    """The handler of a model observed as ``data['y']``, or through a streaming engine when there is no ``data``: the
    checks these models share, then ``run(model, ctx, y, mask=..., inputs=..., predict=..., horizon=..., **keywords)``
    under the guard."""
    def handler(model, **kw):
        data = kw["data"]
        if isinstance(model, _WISHART_LGSSMS):
            if data is not None and "u" in data:
                raise NotImplementedError("data['u']: input sequences on the Wishart-precision LGSSM are outside the "
                                          "batched hot path (a constant offset is model.u)")
            if isinstance(kw["returnvars"], dict) and isinstance(kw["returnvars"].get("x"), KeepEach):
                raise NotImplementedError("returnvars: q(x) is kept for the last iteration only (KeepLast) on the "
                                          "batched path")
            if data is None:
                raise ValueError("the Wishart-precision LGSSM needs `data` (it has no streaming form)")
        horizon = getattr(model, "horizon", 0) if isinstance(model, linear_gaussian_ssm_smoothing) else 0
        if isinstance(model, linear_gaussian_ssm_filtering) and horizon:
            raise NotImplementedError("horizon > 0 belongs to the smoothing LGSSM")
        predict = None
        if kw["predictvars"] is not None or horizon > 0:
            predict = _predict_keys(kw["predictvars"] if kw["predictvars"] is not None else {}, model, data)
        if data is None:
            if kw["datastream"] is None and kw["autoupdates"] is None:
                raise ValueError("either `data` or `datastream` (or `autoupdates` for a push-driven engine) is "
                                 "required")
            if kw["batch"] is None:
                raise ValueError("streaming inference needs `batch` (number of lock-step datastreams)")
            from .streaming import RxInferenceEngine
            return RxInferenceEngine(kw["context"] or default_context(), model, batch=kw["batch"],
                                     iterations=kw["iterations"], keephistory=kw["keephistory"],
                                     historyvars=kw["historyvars"], free_energy=kw["free_energy"],
                                     datastream=kw["datastream"], autostart=kw["autostart"],
                                     cov_shared_out=kw["cov_shared_out"])
        if "y" not in data:
            raise KeyError("data must contain the observations under key 'y'")   # reference: missing data key error
        y = data["y"]
        # known per-step inputs x[t] ~ A x[t-1] + u[t]: data["u"] is a host [T(+H), d] sequence shared by every chain or
        # a CUDA [T(+H), d, batch] tensor (one sequence per chain)
        inputs = data.get("u")
        if inputs is not None and getattr(model, "u", None) is not None:
            raise ValueError("the model has a constant offset u and data carries an input sequence 'u': fold the "
                             "constant into the sequence")
        if inputs is not None and not isinstance(model, linear_gaussian_ssm_smoothing):
            raise NotImplementedError(f"data['u']: input sequences belong to the LGSSM, not {type(model).__name__}")
        if inputs is not None and horizon > 0 and inputs.shape[0] != y.shape[0] + horizon:
            raise ValueError(f"data['u'] needs T + horizon = {y.shape[0] + horizon} rows (the forecasts use the inputs "
                             f"of the forecast steps), got {inputs.shape[0]}")
        return lambda ctx: run(model, ctx, y, mask=data.get("ymask"), inputs=inputs, predict=predict, horizon=horizon,
                               **kw)
    return handler


@_series
def _infer_lgssm_filtering(model, ctx, y, *, mask, inputs, free_energy, cov_shared_out, **_):
    r = ctx.lgssm(y, model.A, model.B, model.P, model.Q, model.x0[0], model.x0[1], u=model.u, inputs=inputs,
                  smooth=False, mask=mask, want_evidence=free_energy, per_chain_model=model.per_chain,
                  transition_first=True, cov_shared_out=cov_shared_out)
    q = MvNormalMeanCovariance(r["mean"], r["cov"])
    return InferenceResult(posteriors={}, history={"x_t": q}, free_energy=r["neg_log_evidence"], model=model)


@_series
def _infer_lgssm_smoothing(model, ctx, y, *, mask, inputs, predict, horizon, iterations, free_energy, cov_shared_out,
                           **_):
    if iterations not in (None, 1):
        raise NotImplementedError("iterations > 1 on a tree-structured BP model is a no-op in the reference; "
                                  "KeepEach() results are outside the hot path")
    if predict is not None:
        r = ctx.lgssm_predict(y, model.A, model.B, model.P, model.Q, model.x0[0], model.x0[1], horizon=horizon,
                              u=model.u, inputs=inputs, mask=mask, want_evidence=free_energy,
                              per_chain_model=model.per_chain, cov_shared_out=cov_shared_out,
                              transition_first=model.prior_on_previous_state, want_status=True)
        # e.g. a chain whose D_t = Q - B S_s B' is not SPD has no usable prediction
        _raise_flagged(r["status"], "predictions: ", " (NOT_SPD: Q - B S_s B' is not SPD, the observations dominate "
                                                     "beyond the fp32 posterior covariances)")
        T = y.shape[0]
        mean, cov = r["mean"], r["cov"]
        if horizon > 0:          # posteriors["x"] covers x[1..T+H], as model_1's x covers n + 2 states
            mean, cov = torch.cat([mean, r["fc_mean"]]), torch.cat([cov, r["fc_cov"]])
        preds = {}
        if "y" in predict:
            preds["y"] = MvNormalMeanCovariance(r["pred_mean"][:T], r["pred_cov"][:T])
        if "o" in predict:
            preds["o"] = MvNormalMeanCovariance(r["pred_mean"][T:], r["pred_cov"][T:])
        return InferenceResult(posteriors={"x": MvNormalMeanCovariance(mean, cov)}, predictions=preds,
                               free_energy=r["neg_log_evidence"], model=model)
    r = ctx.lgssm(y, model.A, model.B, model.P, model.Q, model.x0[0], model.x0[1], u=model.u, inputs=inputs,
                  smooth=True, mask=mask, want_evidence=free_energy, per_chain_model=model.per_chain,
                  cov_shared_out=cov_shared_out, transition_first=model.prior_on_previous_state)
    return InferenceResult(posteriors={"x": MvNormalMeanCovariance(r["mean"], r["cov"])},
                           free_energy=r["neg_log_evidence"], model=model)


@_series
def _infer_hgf(model, ctx, y, *, iterations, free_energy, **_):
    out = ctx.hgf_filter(y, iters=iterations or 1, kappa=model.real_k, omega=model.real_w,
                         z_variance=model.z_variance, y_variance=model.y_variance, init=model.init,
                         want_free_energy=bool(free_energy))
    fe = None
    if free_energy:      # free_energy_history of the streaming engine: average over the data, per iteration
        out, fe_all = out
        fe = fe_all.mean(dim=0)
    return InferenceResult(posteriors={}, model=model, free_energy=fe,
                           history={"xt": NormalMeanVariance(out[:, 0], out[:, 1]),
                                    "zt": NormalMeanVariance(out[:, 2], out[:, 3])})


@_series
def _infer_kalman_gamma(model, ctx, y, *, iterations, free_energy, **_):
    out, fe = ctx.stream_vmp_gamma(y, iters=iterations or 1, w=model.transition_precision, init=model.init,
                                   want_free_energy=bool(free_energy))
    return InferenceResult(posteriors={}, model=model, free_energy=None if fe is None else fe.mean(dim=0),
                           history={"x_t": NormalMeanVariance(out[:, 0], out[:, 1]),
                                    "τ": GammaShapeRate(out[:, 2], out[:, 3])})


@_series
def _infer_lgssm_gamma(model, ctx, y, *, iterations, free_energy, **_):
    r = ctx.lgssm_vmp_gamma(y, iterations=iterations or 1, a=model.a, v_proc=model.v_proc, prior=model.x0,
                            gamma_prior=model.gamma_prior, init_E_tau=model.init_E_tau,
                            want_free_energy=bool(free_energy))
    return InferenceResult(posteriors={"x": NormalMeanVariance(r["mean"], r["var"]),
                                       "τ": GammaShapeRate(r["shape"], r["rate"])}, model=model,
                           free_energy=r["free_energy"])


@_series
def _infer_wishart_precision(model, ctx, y, *, mask, iterations, free_energy, **_):
    r = ctx.lgssm_vmp_wishart(y, model.A, model.B, model.P, model.x0[0], model.x0[1], iterations=iterations or 1,
                              w_prior=(model.w_prior.df, model.w_prior.inv_scale()), init_E_W=model.w_init.mean(),
                              u=model.u, mask=mask, transition_first=model.prior_on_previous_state,
                              want_free_energy=bool(free_energy))
    _raise_flagged(r["status"])
    # returnvars of the reference's call under `iterations`: x = KeepLast() here, w = KeepEach() (iteration axis)
    return InferenceResult(posteriors={"x": MvNormalMeanCovariance(r["mean"], r["cov"]),
                                       "w": WishartFast(r["df"], r["inv_scale"])},
                           model=model, free_energy=r["free_energy"])


@_series
def _infer_wishart_noise(model, ctx, y, *, mask, iterations, free_energy, **_):
    r = ctx.lgssm_vmp_noise(y, model.A, model.B, model.x0[0], model.x0[1], **_noise_kwargs(model), u=model.u,
                            mask=mask, transition_first=model.prior_on_previous_state,
                            iterations=iterations or 1, want_free_energy=bool(free_energy))
    _raise_flagged(r["status"])
    # x = KeepLast(), w_p / w_q = KeepEach() (leading iteration axis) for the learned precisions
    return InferenceResult(posteriors={"x": MvNormalMeanCovariance(r["mean"], r["cov"]), **_noise_posteriors(r)},
                           model=model, free_energy=r["free_energy"])


@_series
def _infer_continuous_transition(model, ctx, y, *, mask, iterations, free_energy, **_):
    kw = _noise_kwargs(model)
    if model.a_init is None:
        raise ValueError("a_init: q(a) needs an initial (mean, covariance) (an uninformed q(a) makes the first "
                         "sweep meaningless)")
    d = np.asarray(model.x0[1]).shape[-1]
    pm = vec_order(d)
    rowmajor = lambda mc: (np.asarray(mc[0], np.float64).reshape(-1)[pm],
                           np.asarray(mc[1], np.float64)[np.ix_(pm, pm)])
    r = ctx.lgssm_vmp_transition(y, model.B, model.x0[0], model.x0[1], a_prior=rowmajor(model.a_prior),
                                 a_init=rowmajor(model.a_init), **kw, u=model.u, mask=mask,
                                 transition_first=model.prior_on_previous_state, iterations=iterations or 1,
                                 want_free_energy=bool(free_energy))
    _raise_flagged(r["status"])
    # x = KeepLast(); a, w_p / w_q = KeepEach() (leading iteration axis); a over vec(A) in column-major order
    pt = torch.as_tensor(pm, device=r["a_mean"].device)
    its_, nb = r["a_mean"].shape[0], r["a_mean"].shape[-1]
    a_mu = r["a_mean"].reshape(its_, d * d, nb)[:, pt]
    a_S = r["a_cov"][:, pt][:, :, pt]
    return InferenceResult(posteriors={"x": MvNormalMeanCovariance(r["mean"], r["cov"]),
                                       "a": MvNormalMeanCovariance(a_mu, a_S), **_noise_posteriors(r)},
                           model=model, free_energy=r["free_energy"])


@_series
def _infer_mixture(model, ctx, y, *, constraints, initialization, iterations, free_energy, returnvars, **_):
    check_mean_field(constraints)
    each = _kept_each("gaussian_mixture", returnvars, ("s", "m", "w"), by_name=False)
    arr = gaussian_mixture_arrays(model, initialization)
    yy = y[:, None] if y.dim() == 2 else y          # univariate data may come as [N, batch]
    if yy.shape[1] != arr["mu0"].shape[1]:
        raise ValueError(f"data['y'] has d = {yy.shape[1]}, the model's means d = {arr['mu0'].shape[1]}")
    r = ctx.gmm_vmp(yy.contiguous(), *(arr[k] for k in ("alpha0", "mu0", "V0", "nu0", "S0", "alpha_init", "m_init",
                                                         "Vm_init", "nu_init", "S_init")),
                    iterations=iterations or 1, want_free_energy=bool(free_energy), want_z=True, keep_each=bool(each))
    _raise_flagged(r["status"], "gaussian_mixture: ", " (NOT_SPD: an update met a non-SPD matrix)")
    al = r["hist_alpha" if each else "alpha"]       # KeepEach: a leading iteration axis on every posterior
    post = {"s": Beta(al[..., 0, :], al[..., 1, :]) if arr["univariate"] else Dirichlet(al)}
    post["m"], post["w"] = _component_posteriors(r, each, arr["univariate"])
    post["z"] = Categorical(r["z_prob"])
    return InferenceResult(posteriors=post, model=model, free_energy=r["free_energy"])


@_series
def _infer_lar(model, ctx, y, *, iterations, free_energy, **_):
    yy = y[:, 0] if y.dim() == 3 else y
    r = ctx.lar_vmp(yy.contiguous(), model.order, model.tau, iterations=iterations or 1, gamma_prior=model.gamma_prior,
                    theta_prior_precision=model.theta_prior_precision, x0_prior_precision=model.x0_prior_precision,
                    init_gamma=model.init_gamma, init_theta_precision=model.init_theta_precision,
                    want_free_energy=bool(free_energy))
    # returnvars of the reference's call: x = KeepLast(), gamma / theta = KeepEach() (leading iteration axis)
    return InferenceResult(posteriors={"x": MvNormalMeanCovariance(r["x_mean"], r["x_cov"]),
                                       "γ": GammaShapeRate(r["gamma_shape"], r["gamma_rate"]),
                                       "θ": MvNormalMeanCovariance(r["theta_mean"], r["theta_cov"])},
                           model=model, free_energy=r["free_energy"])


@_series
def _infer_unrecognised(model, ctx, y, **_):
    raise NotImplementedError(f"model pattern {type(model).__name__} is not on the batched hot path")


class _Model(NamedTuple):
    """What ``infer`` knows of one model besides its handler: the refusals it states once for the model."""
    handler: object
    takes_constraints: bool = False          # `constraints` is a keyword of the model (else it is refused)
    check_constraints: object = None         # checked before every other refusal (the mixture checks its own, guarded)
    refuses: tuple = ()                      # streaming keywords refused with NotImplementedError
    refusal_note: str = ""                   # appended to that refusal
    predictions_of: str = None               # predictvars refused: "predictions of <this> are outside ..."
    whole_data: str = None                   # datastream refused: "<model> <this>"
    context_guarded: bool = False            # the context lookup is under the catch_exception guard
    takes_meta: bool = False                 # `meta` is a keyword of the model (its Delta nodes' approximations)


_STREAMING = ("autoupdates", "keephistory", "historyvars", "batch", "cov_shared_out")
_WISHART_LGSSM = "the Wishart-precision LGSSM"

_MODELS = {
    linear_gaussian_ssm_filtering: _Model(_infer_lgssm_filtering),
    linear_gaussian_ssm_smoothing: _Model(_infer_lgssm_smoothing),
    hgf: _Model(_infer_hgf),
    kalman_gamma_streaming: _Model(_infer_kalman_gamma),
    univariate_lgssm_gamma_precision: _Model(_infer_lgssm_gamma),
    linear_gaussian_ssm_wishart_precision: _Model(_infer_wishart_precision, predictions_of=_WISHART_LGSSM),
    linear_gaussian_ssm_wishart_noise: _Model(_infer_wishart_noise, predictions_of=_WISHART_LGSSM),
    linear_gaussian_ssm_continuous_transition: _Model(_infer_continuous_transition, predictions_of=_WISHART_LGSSM),
    gaussian_mixture: _Model(_infer_mixture, takes_constraints=True),
    latent_autoregressive: _Model(_infer_lar),
    hidden_markov_model: _Model(_infer_hmm, takes_constraints=True, check_constraints=check_hmm_constraints,
                                predictions_of="the hidden Markov model", context_guarded=True),
    gaussian_hidden_markov_model: _Model(_infer_hmm_gauss, takes_constraints=True,
                                         check_constraints=_check_gaussian_hmm_constraints,
                                         predictions_of="the Gaussian hidden Markov model",
                                         whole_data="runs over whole series: pass data = {'y': [T, d, batch]} "
                                                    "(no datastream)", context_guarded=True),
    hgf_offline: _Model(_infer_hgf_offline, takes_constraints=True, check_constraints=_check_hgf_offline_constraints,
                        predictions_of="the HGF",
                        whole_data="runs over whole series: pass data = {'y': [T, batch]} (no datastream)",
                        context_guarded=True),
    binomial_regression: _Model(_infer_binomial, refuses=_STREAMING, predictions_of="y",
                                whole_data="runs over whole data sets: pass data = {'X', 'y', 'n_trials'} "
                                           "(no datastream)", context_guarded=True),
    multinomial_regression: _Model(_infer_multinomial, refuses=_STREAMING,
                                   refusal_note=" (the online form is multinomial_regression_online)",
                                   predictions_of="y",
                                   whole_data="runs over whole data sets: pass data = {'y'} (the online form is "
                                              "multinomial_regression_online)", context_guarded=True),
    multinomial_regression_online: _Model(_infer_multinomial_online, refuses=("cov_shared_out",)),
    gamma_mixture: _Model(_infer_gamma_mixture, takes_constraints=True, check_constraints=_check_gamma_mixture_constraints,
                          refuses=_STREAMING, predictions_of="y",
                          whole_data="runs over whole data sets: pass data = {'y': [N, batch]} (no datastream)",
                          context_guarded=True),
    nonlinear_gaussian_ssm_smoothing: _Model(_infer_delta, takes_meta=True, refuses=_STREAMING,
                                             refusal_note=" (the streaming form is nonlinear_gaussian_ssm_filtering)"),
    nonlinear_gaussian_ssm_filtering: _Model(_infer_delta, takes_meta=True, refuses=("cov_shared_out",)),
    nonlinear_gamma_streaming: _Model(_infer_delta, takes_meta=True, takes_constraints=True,
                                      check_constraints=_check_delta_constraints, refuses=("cov_shared_out",)),
}
_UNRECOGNISED = _Model(_infer_unrecognised)


def infer(*, model, iterations=None, free_energy=False, returnvars=None, options=None,
          initialization=None, autoupdates=None, keephistory=None, historyvars=None,
          catch_exception=False, showprogress=False, session=None, warn=True, allow_node_contraction=False,
          context: Context | None = None, cov_shared_out=False, data=None, datastream=None, autostart=True,
          batch=None, predictvars=None, **kwargs):
    """Batched ``infer``.  ``data = {"y": tensor[T, m, batch]}`` (CUDA fp32, or CPU for the
    host-staged path).  Returns ``posteriors["x"]`` as a batched ``MvNormalMeanCovariance``.

    With ``datastream=`` (an iterable of time-chunks, or ``None`` + ``autoupdates`` for a push-driven
    engine) the call returns an ``RxInferenceEngine`` (streaming.py), as the reference does when
    ``autoupdates`` is given (/root/reference/src/inference/inference.jl:577-733 dispatch)."""
    spec = next((_MODELS[t] for t in type(model).__mro__ if t in _MODELS), _UNRECOGNISED)
    constraints = kwargs.pop("constraints", None) if spec.takes_constraints else None
    meta = kwargs.pop("meta", None) if spec.takes_meta else None
    for k in kwargs:
        if k in _UNSUPPORTED:
            raise NotImplementedError(
                f"infer(..., {k}=...) needs per-message machinery outside the batched hot path; "
                "run this call through stock ReactiveMP")
        raise TypeError(f"infer() got an unexpected keyword argument '{k}'")
    if options:
        bad = set(options) - {"limit_stack_depth", "warn"}   # limit_stack_depth is moot: the schedule is a fused sweep
        if bad:
            raise NotImplementedError(f"options {sorted(bad)} are outside the batched hot path")
    if data is not None and datastream is not None:
        raise ValueError("`data` and `datastream` are mutually exclusive")    # reference: inference.jl argument check
    if spec.check_constraints is not None:
        spec.check_constraints(constraints)
    given = dict(autoupdates=autoupdates is not None, keephistory=keephistory is not None,
                 historyvars=historyvars is not None, batch=batch is not None, cov_shared_out=bool(cov_shared_out))
    if any(given[k] for k in spec.refuses):
        names = " and ".join(filter(None, (", ".join(spec.refuses[:-1]), spec.refuses[-1])))
        raise NotImplementedError(f"{type(model).__name__}: {names} {'are' if len(spec.refuses) > 1 else 'is'} outside "
                                  f"the batched hot path{spec.refusal_note}")
    if spec.predictions_of is not None and predictvars is not None:
        raise NotImplementedError(f"predictvars: predictions of {spec.predictions_of} are outside the batched hot path")
    if spec.whole_data is not None and (datastream is not None or data is None):
        raise NotImplementedError(f"{type(model).__name__} {spec.whole_data}")
    run = spec.handler(model, data=data, constraints=constraints, initialization=initialization, iterations=iterations,
                       free_energy=free_energy, returnvars=returnvars, predictvars=predictvars, datastream=datastream,
                       autoupdates=autoupdates, keephistory=keephistory, historyvars=historyvars, autostart=autostart,
                       batch=batch, cov_shared_out=cov_shared_out, context=context, meta=meta)
    if not callable(run):
        return run                                   # a streaming engine
    if not spec.context_guarded:
        context = context or default_context()       # looked up before the guard, so a missing device raises
    try:
        return run(context or default_context())
    except Exception as e:           # reference: catch_exception=true returns a partial result with .error
        if catch_exception:
            return InferenceResult(posteriors={}, model=model, error=e)
        raise
