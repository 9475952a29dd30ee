"""Batched message / marginal containers named after the reference's distribution types
(ExponentialFamily.jl, aliases at /root/reference/src/model/graphppl.jl:340-423).

Every container holds structure-of-arrays CUDA tensors with the batch axis innermost, the layout
of the C ABI.  ``mean`` / ``cov`` / ``var`` / ``mean_cov`` mirror the accessors user code calls
on ``posteriors[:x]`` (e.g. /root/reference/test/models/statespace/mlgssm_test.jl:121-126).
"""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np
import torch


@dataclass
class PointMass:
    """Constant / datum (factorised out by default, /root/reference/src/model/model.jl:198,222), or a marginal under a
    point-mass form constraint."""
    value: object

    def mean(self):
        return self.value


@dataclass
class MvNormalMeanCovariance:
    mu: torch.Tensor       # [..., d, n]
    Sigma: torch.Tensor    # [..., d, d, n]  (or [..., d, d] when shared across the batch)

    def mean(self):
        return self.mu

    def cov(self):
        return self.Sigma

    def var(self):
        return torch.diagonal(self.Sigma, dim1=-3, dim2=-2) if self.Sigma.dim() == self.mu.dim() + 1 \
            else torch.diagonal(self.Sigma, dim1=-2, dim2=-1)

    def mean_cov(self):
        return self.mu, self.Sigma


@dataclass
class MvNormalWeightedMeanPrecision:
    xi: torch.Tensor
    W: torch.Tensor

    def weightedmean_precision(self):
        return self.xi, self.W


@dataclass
class NormalMeanVariance:
    m: torch.Tensor
    v: torch.Tensor

    def mean(self):
        return self.m

    def var(self):
        return self.v

    def mean_var(self):
        return self.m, self.v


@dataclass
class GammaShapeRate:
    a: torch.Tensor
    b: torch.Tensor

    def mean(self):
        return self.a / self.b

    def shape(self):
        return self.a

    def rate(self):
        return self.b


@dataclass
class WishartFast:
    """Wishart in the (df, INVERSE scale) parametrisation ReactiveMP uses for messages (``WishartFast``):
    ``df[n]``, ``invS[d, d, n]``; products are additions."""
    df: torch.Tensor
    invS: torch.Tensor


@dataclass
class Wishart:
    """``Wishart(df, scale)`` as a model is written (a prior or an initial marginal): host ``scale[m, m]``."""
    df: float
    scale: object

    def inv_scale(self):
        return np.linalg.inv(np.asarray(self.scale, dtype=np.float64))

    def mean(self):
        return float(self.df) * np.asarray(self.scale, dtype=np.float64)


@dataclass
class Dirichlet:
    """``Dirichlet(alpha)``: ``alpha[K]`` (host, a prior or an initial marginal) or ``alpha[..., K, n]`` (posteriors)."""
    alpha: object

    def mean(self):
        a = self.alpha
        return a / a.sum(dim=-2, keepdim=True) if isinstance(a, torch.Tensor) else np.asarray(a, np.float64) / np.sum(a)


@dataclass
class Beta:
    """``Beta(a, b)`` = ``Dirichlet([a, b])``: the weight of the first of two components."""
    a: object
    b: object

    def mean(self):
        return self.a / (self.a + self.b)


@dataclass
class DirichletCollection:
    """``DirichletCollection(alpha)``: a matrix whose columns are independent Dirichlets (column j is the distribution
    conditioned on state j).  ``alpha[R, C]`` (host, a prior or an initial marginal) or ``alpha[..., R, C, n]``
    (posteriors)."""
    alpha: object

    def mean(self):
        a = self.alpha
        if isinstance(a, torch.Tensor):
            return a / a.sum(dim=-3, keepdim=True)
        a = np.asarray(a, np.float64)
        return a / a.sum(axis=0, keepdims=True)


@dataclass
class Categorical:
    """``Categorical(p)``: ``p[..., K, n]``."""
    p: torch.Tensor

    def probvec(self):
        return self.p


def vague(kind, like=None):
    """``vague(NormalMeanVariance)`` = N(0, 1e12); ``vague(GammaShapeRate)`` = Gamma(1, 1e-12)
    (TinyHugeNumbers, upstream); ``vague(Beta)`` = Beta(1, 1); ``vague(Dirichlet, K)`` = Dirichlet(ones(K));
    ``vague(DirichletCollection, (R, C))`` = DirichletCollection(ones(R, C)); ``vague(Categorical, K)`` = uniform.
    With a tensor ``like`` the parameters are tensors shaped like it, else host floats."""
    if kind is Beta:
        return Beta(1.0, 1.0)
    if kind is Dirichlet:
        if not isinstance(like, (int, np.integer)) or like < 1:
            raise TypeError("vague(Dirichlet, K) needs the number of components K")
        return Dirichlet(np.ones(int(like)))
    if kind is DirichletCollection:
        if not (isinstance(like, tuple) and len(like) == 2 and all(isinstance(n, (int, np.integer)) and n >= 1 for n in like)):
            raise TypeError("vague(DirichletCollection, (R, C)) needs the matrix shape")
        return DirichletCollection(np.ones(like))
    if kind is Categorical:
        if not isinstance(like, (int, np.integer)) or like < 1:
            raise TypeError("vague(Categorical, K) needs the number of categories K")
        return Categorical(np.full(int(like), 1.0 / int(like)))
    if like is None:
        if kind is NormalMeanVariance:
            return NormalMeanVariance(0.0, 1e12)
        if kind is GammaShapeRate:
            return GammaShapeRate(1.0, 1e-12)
        raise TypeError(kind)
    if kind is NormalMeanVariance:
        return NormalMeanVariance(torch.zeros_like(like), torch.full_like(like, 1e12))
    if kind is GammaShapeRate:
        return GammaShapeRate(torch.ones_like(like), torch.full_like(like, 1e-12))
    raise TypeError(kind)
