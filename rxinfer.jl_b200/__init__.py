"""rxinfer.jl_b200 -- H100-native (sm_90a) Gaussian message-passing hot path of RxInfer.jl.

Contents: ``csrc/`` (CUDA kernels + the C ABI of ``librxgauss.so``, header in ``include/rxgauss.h``),
this host-side mirror of the reference interface (``infer``, ``call_rule``, distribution
containers) over ctypes, and ``julia/RxGaussB200.jl`` (the ccall shim a maintainer would add).
Importing the package does NOT load the CUDA library; the first compute call does, and fails
loudly if it is missing or no GPU is present -- there is no CPU fallback.
"""
from . import _lib
from ._lib import RxGaussError
from .distributions import (Beta, Categorical, Dirichlet, DirichletCollection, GammaShapeRate, MvNormalMeanCovariance,
                            MvNormalWeightedMeanPrecision, NormalMeanVariance, PointMass, Wishart, WishartFast, vague)


def __getattr__(name):   # lazy: these import torch
    if name in ("Context", "comm_unique_id"):
        from . import context
        return getattr(context, name)
    if name in ("infer", "InferenceResult", "linear_gaussian_ssm_smoothing", "linear_gaussian_ssm_filtering",
                "hgf", "univariate_lgssm_gamma_precision", "kalman_gamma_streaming", "latent_autoregressive",
                "linear_gaussian_ssm_wishart_precision", "linear_gaussian_ssm_wishart_noise",
                "linear_gaussian_ssm_continuous_transition", "gaussian_mixture", "MeanField", "BetheFactorization",
                "hidden_markov_model", "HMMConstraints", "hgf_offline", "gaussian_hidden_markov_model",
                "GaussianHMMConstraints", "binomial_regression", "multinomial_regression",
                "multinomial_regression_online", "CudaFunction", "Linearization", "Unscented",
                "nonlinear_gaussian_ssm_smoothing", "nonlinear_gaussian_ssm_filtering", "nonlinear_gamma_streaming",
                "gamma_mixture", "GammaMixtureConstraints", "default_context",
                "KeepLast", "KeepEach"):
        from . import inference
        return getattr(inference, name)
    if name in ("call_rule", "prod", "RuleMethodError"):
        from . import rules
        return getattr(rules, name)
    if name == "RxInferenceEngine":
        from . import streaming
        return streaming.RxInferenceEngine
    if name == "sharding":
        import importlib
        return importlib.import_module(".sharding", __name__)
    raise AttributeError(name)
