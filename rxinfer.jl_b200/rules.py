"""``call_rule``: the Python mirror of ``@call_rule Node(:edge, Marginalisation)(m_a = ..., q_b = ...)``
(/root/reference/test/inference/inference_tests.jl:547-585), dispatching to the batched CUDA rule
kernels.  Same node / edge / message names as the reference's ``@rule`` signatures
(SURVEY.md section 8a); anything outside the Gaussian hot path raises ``RuleMethodError`` exactly
like a missing ``@rule`` method would in ReactiveMP.
"""
from __future__ import annotations

from .distributions import (GammaShapeRate, MvNormalMeanCovariance, MvNormalWeightedMeanPrecision,
                            NormalMeanVariance, PointMass, WishartFast)


class RuleMethodError(NotImplementedError):
    pass


def _meancov(msg):
    """(mu [d, n], Sigma [d, d, n]) of a mean-covariance message: a covariance [d, d] shared by the batch (the form
    ``MvNormalMeanCovariance`` documents) is expanded to one per message, the layout every rule kernel reads."""
    mu, S = msg.mu, msg.Sigma
    if S.dim() == 2 and mu.dim() == 2:
        S = S.unsqueeze(-1).expand(*S.shape, mu.shape[-1]).contiguous()
    return mu, S


def _mc(ctx, msg):
    """mean_cov(msg): converts a (xi, W) message with one cholinv, like the reference."""
    if isinstance(msg, MvNormalMeanCovariance):
        return _meancov(msg)
    if isinstance(msg, MvNormalWeightedMeanPrecision):
        mu, S, _ = ctx.wmp_to_meancov(msg.xi, msg.W)
        return mu, S
    raise RuleMethodError(f"expected a multivariate normal message, got {type(msg).__name__}")


def _wmp(ctx, msg):
    if isinstance(msg, MvNormalWeightedMeanPrecision):
        return msg.xi, msg.W
    xi, W, _ = ctx.meancov_to_wmp(*_meancov(msg))
    return xi, W


def call_rule(ctx, node: str, edge: str, **kw):
    key = (node, edge, tuple(sorted(kw)))
    if node == "MvNormalMeanCovariance":
        if edge == "out" and "m_μ" in kw and "q_Σ" in kw:
            mu, S = _mc(ctx, kw["m_μ"])
            return MvNormalMeanCovariance(*ctx.rule_add_cov(mu, S, kw["q_Σ"].value, "out"))
        if edge == "μ" and "m_out" in kw and "q_Σ" in kw:
            mu, S = _mc(ctx, kw["m_out"])
            return MvNormalMeanCovariance(*ctx.rule_add_cov(mu, S, kw["q_Σ"].value, "mean"))
        if edge == "μ" and "q_out" in kw and "q_Σ" in kw and isinstance(kw["q_out"], PointMass):
            return MvNormalMeanCovariance(*ctx.rule_mean_from_data(kw["q_out"].value, kw["q_Σ"].value))
    if node == "*":
        if edge == "out" and "m_A" in kw and "m_in" in kw:
            mu, S = _mc(ctx, kw["m_in"])
            return MvNormalMeanCovariance(*ctx.rule_mul_out(kw["m_A"].value, mu, S))
        if edge == "in" and "m_out" in kw and "m_A" in kw:
            if kw.get("meta") is not None:
                raise RuleMethodError("`*`(:in) with a correction meta is outside the hot path")
            mu, S = _mc(ctx, kw["m_out"])
            xi, W, _ = ctx.rule_mul_in(kw["m_A"].value, mu, S)
            return MvNormalWeightedMeanPrecision(xi, W)
    if node == "+":
        if edge == "out":
            a, b = _mc(ctx, kw["m_in1"]), _mc(ctx, kw["m_in2"])
            return MvNormalMeanCovariance(*ctx.rule_add_out(*a, *b))
        if edge in ("in1", "in2"):
            other = "m_in2" if edge == "in1" else "m_in1"
            a, b = _mc(ctx, kw["m_out"]), _mc(ctx, kw[other])
            return MvNormalMeanCovariance(*ctx.rule_add_in(*a, *b))
    if node == "NormalMeanPrecision":
        if edge == "τ" and "q_out" in kw and "q_μ" in kw:
            (mo, vo), (mm, vm) = kw["q_out"].mean_var(), kw["q_μ"].mean_var()
            return GammaShapeRate(*ctx.rule_normal_precision_tau(mo, vo, mm, vm))
        if edge == "τ" and "q_out_μ" in kw:
            # structured: q(out, mu) jointly Gaussian (MvNormalMeanCovariance with d = 2)
            return GammaShapeRate(*ctx.rule_normal_precision_tau_joint(*_mc(ctx, kw["q_out_μ"])))
        if edge == "out" and "q_τ" in kw and "m_μ" in kw:
            # (m_μ::Normal, q_τ): belief-propagation message on the mean edge -> N(m_μ, v_μ + 1/E[τ])
            src = kw["m_μ"]
            return NormalMeanVariance(*ctx.rule_normal_precision_out(src.m, src.v, kw["q_τ"].a, kw["q_τ"].b))
        if edge == "out" and "q_τ" in kw and "q_μ" in kw:
            # (q_μ::Any, q_τ::Any): mean-field -> NormalMeanPrecision(mean(q_μ), mean(q_τ)): variance 1/E[τ] ONLY,
            # var(q_μ) does not enter (same kernel with v_μ = 0)
            m, _ = kw["q_μ"].mean_var()
            return NormalMeanVariance(*ctx.rule_normal_precision_out(m, m.new_zeros(m.shape), kw["q_τ"].a, kw["q_τ"].b))
    if node == "MvNormalMeanPrecision":
        if edge == "Λ" and "q_out" in kw and "q_μ" in kw:
            (mo, Vo), (mm, Vm) = _mc(ctx, kw["q_out"]), _mc(ctx, kw["q_μ"])
            return WishartFast(*ctx.rule_mvnormal_precision_lambda(mo, Vo, mm, Vm))
    if node == "GCV":
        k, w = float(kw["q_κ"].value), float(kw["q_ω"].value)
        if edge in ("y", "x"):
            src = kw["m_x"] if edge == "y" else kw["m_y"]
            return NormalMeanVariance(*ctx.rule_gcv_out(src.m, src.v, kw["q_z"].m, kw["q_z"].v, k, w))
    raise RuleMethodError(f"no batched rule for {key}; route this node to stock ReactiveMP")


def prod(ctx, left, right):
    """``BayesBase.prod(GenericProd(), left, right)`` for the Gaussian / Gamma family."""
    if isinstance(left, GammaShapeRate) and isinstance(right, GammaShapeRate):
        return GammaShapeRate(*ctx.prod_gamma(left.a, left.b, right.a, right.b))
    if isinstance(left, WishartFast) and isinstance(right, WishartFast):
        return WishartFast(*ctx.prod_wishart(left.df, left.invS, right.df, right.invS))
    if isinstance(left, NormalMeanVariance) and isinstance(right, NormalMeanVariance):
        return NormalMeanVariance(*ctx.prod_normal(left.m, left.v, right.m, right.v))
    l, r = _wmp(ctx, left), _wmp(ctx, right)
    return MvNormalWeightedMeanPrecision(*ctx.prod_gaussian(*l, *r))
