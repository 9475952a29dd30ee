"""``RxInferenceEngine``: the streaming half of ``infer()`` (/root/reference/src/inference/streaming.jl:16-140
result object, :186-300 start/stop, :344-430 the per-datum executor, :536-845 ``streaming_inference``),
mirrored for ``batch`` independent datastreams that tick in lock-step.

The reference re-runs a ONE-step factor graph per datum and feeds ``q(x_t)`` back into the next prior through
``@autoupdates`` (src/inference/autoupdates.jl:614-659).  Here the datastream delivers time-CHUNKS
``y[Tc, m, batch]`` (any Tc >= 1, may vary from chunk to chunk); every chunk is one fused filtering sweep on
the GPU (``rxg_lgssm_filter_chunk_f32`` / ``rxg_hgf_filter_chunk_f32``) and the engine holds the autoupdate
carry between chunks.  ``keephistory`` / ``historyvars`` follow the reference: a circular buffer of the last
``keephistory`` marginals per history variable (``KeepLast`` per datum is the only strategy on a BP model).
"""
from __future__ import annotations

import numpy as np
import torch

from .distributions import GammaShapeRate, MvNormalMeanCovariance, NormalMeanVariance


class RxInferenceEngine:
    """Created by ``infer(model=..., datastream=..., autoupdates=..., keephistory=...)``.

    ``datastream``: an iterable of chunks (CUDA fp32 tensors ``[Tc, m, batch]``, or ``[Tc, batch]`` for the
    HGF; an LGSSM chunk may also be ``{"y": ..., "u": ...}`` with the chunk's known inputs), or ``None`` for a push-driven engine (``engine.push(chunk)``; the reference's
    ``Subject``-style datastream).  ``autostart=True`` consumes an iterable datastream immediately."""

    def __init__(self, ctx, model, *, batch, iterations=1, keephistory=None, historyvars=None, free_energy=False,
                 datastream=None, autostart=True, cov_shared_out=False, initialization=None, meta=None):
        from . import inference as I
        self.ctx, self.model, self.batch = ctx, model, int(batch)
        self.iterations = int(iterations or 1)
        self.keephistory = keephistory
        self.free_energy_enabled = bool(free_energy)
        self.cov_shared_out = cov_shared_out
        self.datastream = datastream
        self.is_running = self.is_completed = self.is_errored = False
        self.error = None
        self.ticks = 0                       # data consumed so far (per stream)
        self._hist: dict[str, list] = {}
        self._fe: list = []
        if isinstance(model, I.hgf):
            self._kind = "hgf"
            names = ("xt", "zt")
            self._carry = None               # out[-1] of the previous chunk, [4, batch]
        elif isinstance(model, I.kalman_gamma_streaming):
            self._kind = "vmpgamma"
            names = ("x_t", "τ")
            self._carry = None
        elif isinstance(model, I.linear_gaussian_ssm_filtering):
            self._kind = "lgssm"
            names = ("x_t",)
            if model.per_chain:
                raise NotImplementedError("streaming chunks need the shared-model gain-table path")
            m0 = torch.as_tensor(np.asarray(model.x0[0], np.float32), device=f"cuda:{ctx.device}")
            self._prev_mean = m0[:, None].expand(-1, self.batch).contiguous()      # q(x_t) initialisation, broadcast
            self._carry_cov = np.ascontiguousarray(np.asarray(model.x0[1], np.float32)).copy()
        elif isinstance(model, (I.nonlinear_gaussian_ssm_filtering, I.nonlinear_gamma_streaming)):
            # the Delta-node filter: the carry q(x) (and q(noise)) is per chain, [d, batch] / [d, d, batch] on the device
            gamma = isinstance(model, I.nonlinear_gamma_streaming)
            self._kind = "delta"
            names = ("state", "noise") if gamma else ("x_t",)
            self._module = I.delta_module(ctx, model, meta)
            mean, cov = model.state0 if gamma else model.x0
            dev = f"cuda:{ctx.device}"
            m0 = torch.as_tensor(np.asarray(mean, np.float32), device=dev)
            S0 = torch.as_tensor(np.asarray(cov, np.float32), device=dev)
            self._mean = m0[:, None].expand(-1, self.batch).contiguous()
            self._cov = S0[:, :, None].expand(-1, -1, self.batch).contiguous()
            self._tau = None
            if gamma:      # Gamma(shape, scale) of the paper -> (shape, rate)
                shape, scale = model.noise0
                self._tau = torch.tensor([[float(shape)], [1.0 / float(scale)]], dtype=torch.float32,
                                         device=dev).expand(-1, self.batch).contiguous()
        elif isinstance(model, I.multinomial_regression_online):
            self._kind = "multinomial"
            names = ("ψ",)
            # the prior of the first datum is the initialization, as the host arrays the C entry takes; the carry
            # q(ψ) = (m, S) is fp64 on the device once the first chunk has run
            self._prior = (np.asarray(initialization.xi, np.float64), np.asarray(initialization.W, np.float64))
            self._carry = None
        else:
            raise NotImplementedError(f"model pattern {type(model).__name__} has no streaming path")
        hv = tuple(historyvars) if historyvars is not None else names
        bad = set(hv) - set(names)
        if bad:
            raise KeyError(f"historyvars {sorted(bad)} are not variables of the model")   # reference: unknown variable error
        self.historyvars = hv
        if autostart and datastream is not None:
            self.start()

    # -------------------------------------------------------------- lifecycle (streaming.jl:186-300)
    def start(self):
        if self.is_completed or self.is_errored:
            raise RuntimeError("The engine has been completed or errored. Cannot start an exhausted engine.")
        if self.is_running:
            return self
        self.is_running = True
        if self.datastream is not None:
            try:
                for chunk in self.datastream:
                    if not self.is_running:
                        break
                    self.push(chunk)
                else:
                    self.is_completed = True
                    self.is_running = False
            except Exception as e:           # reference: the engine records the error and stops (on_error)
                self.is_errored, self.is_running, self.error = True, False, e
                raise
        return self

    def stop(self):
        self.is_running = False
        return self

    # -------------------------------------------------------------- one tick = one chunk (streaming.jl:344-430)
    def push(self, chunk):
        """Consume one chunk; returns the chunk's marginals (dict name -> batched distribution)."""
        inputs = mask = None
        if isinstance(chunk, dict):      # {"y": [Tc, m, batch], "u": the chunk's known inputs ([Tc, d] or [Tc, d, batch])}
            # (the Delta-node engine also takes "ymask": [Tc, batch], 1 = observed)
            if self._kind != "lgssm" and "u" in chunk:
                raise NotImplementedError("input sequences belong to the LGSSM streaming engine")
            chunk, inputs, mask = chunk["y"], chunk.get("u"), chunk.get("ymask")
        if self._kind == "multinomial":
            return self._push_multinomial(chunk)
        if self._kind == "delta":
            return self._push_delta(chunk, mask)
        if self._kind == "lgssm":
            mo = self.model
            r = self.ctx.lgssm_filter_chunk(chunk, mo.A, mo.B, mo.P, mo.Q, self._prev_mean, self._carry_cov, u=mo.u,
                                            inputs=inputs, want_evidence=self.free_energy_enabled,
                                            cov_shared_out=self.cov_shared_out)
            self._prev_mean = r["mean"][-1]              # view into this chunk's output; stays alive through the history or here
            out = {"x_t": MvNormalMeanCovariance(r["mean"], r["cov"])}
            if self.free_energy_enabled:
                self._fe.append(r["neg_log_evidence"])
        elif self._kind == "vmpgamma":
            mo = self.model
            o, fe = self.ctx.stream_vmp_gamma(chunk, iters=self.iterations, w=mo.transition_precision, init=mo.init,
                                              prev=self._carry, want_free_energy=self.free_energy_enabled)
            self._carry = o[-1]
            out = {"x_t": NormalMeanVariance(o[:, 0], o[:, 1]), "τ": GammaShapeRate(o[:, 2], o[:, 3])}
            if self.free_energy_enabled:
                self._fe.append(fe)
        else:
            mo = self.model
            kw = dict(iters=self.iterations, kappa=mo.real_k, omega=mo.real_w, z_variance=mo.z_variance,
                      y_variance=mo.y_variance)
            kw["want_free_energy"] = self.free_energy_enabled
            if self._carry is None:
                o = self.ctx.hgf_filter(chunk, init=mo.init, **kw)
            else:
                o = self.ctx.hgf_filter_chunk(chunk, self._carry, **kw)
            if self.free_energy_enabled:
                o, fe = o
                self._fe.append(fe)
            self._carry = o[-1]
            out = {"xt": NormalMeanVariance(o[:, 0], o[:, 1]), "zt": NormalMeanVariance(o[:, 2], o[:, 3])}
        self.ticks += int(chunk.shape[0])
        self._keep(out)
        return out

    def _push_multinomial(self, chunk):
        """One chunk y[Tc, K, batch] (int32 counts on the device) of the multinomial regression: one
        ``rxg_multinomial_polya_online_f32`` call, the fp64 carry updated in place.  A chunk that flags a chain raises."""
        from .inference import _raise_flagged
        m, S = self._carry if self._carry is not None else (None, None)
        r = self.ctx.multinomial_polya_online(chunk, *self._prior, m=m, S=S, iterations=self.iterations,
                                              want_free_energy=self.free_energy_enabled, keep_mean=bool(self.keephistory),
                                              keep_cov=bool(self.keephistory), in_place=m is not None)
        _raise_flagged(r["status"], "multinomial_regression_online: ", " (BAD_ARG: a negative count; NOT_SPD: a "
                       "non-positive pivot; NAN: a non-finite result)")
        self._carry = (r["m"], r["S"])
        if self.free_energy_enabled:
            self._fe.append(r["free_energy"])
        self.ticks += int(chunk.shape[0])
        out = {"ψ": MvNormalMeanCovariance(r["hist_mean"], r["hist_cov"])} if self.keephistory else {}
        self._keep(out)
        return out

    def _push_delta(self, chunk, mask):
        """One chunk y[Tc, m, batch] (or [Tc, batch] when m = 1) of the Delta-node filter: one
        ``rxg_delta_filter_chunk_f32`` call, the carry updated in place.  A chunk that flags a chain raises."""
        from .inference import _raise_flagged
        mo = self.model
        y = chunk[:, None] if chunk.dim() == 2 else chunk
        d = self._module.d
        P = np.zeros((d, d)) if getattr(mo, "P", None) is None else mo.P
        if self._tau is not None:
            r = self.ctx.delta_filter_chunk(self._module, y.contiguous(), P, self._mean, self._cov,
                                            B=np.asarray(mo.c, np.float64).reshape(1, -1), carry_tau=self._tau,
                                            iters=self.iterations, mask=mask)
        else:
            r = self.ctx.delta_filter_chunk(self._module, y.contiguous(), P, self._mean, self._cov, Q=mo.Q, B=mo.B,
                                            mask=mask)
        _raise_flagged(r["status"], f"{type(mo).__name__}: ", " (NOT_SPD: a predicted or innovation covariance is not "
                                                              "SPD; NAN: a non-finite value)")
        self.ticks += int(y.shape[0])
        out = {("state" if self._tau is not None else "x_t"): MvNormalMeanCovariance(r["mean"], r["cov"])}
        if self._tau is not None:
            out["noise"] = GammaShapeRate(r["tau"][:, 0], r["tau"][:, 1])
        self._keep(out)
        return out

    def _keep(self, out):
        if self.keephistory:
            for name in self.historyvars:
                parts = self._hist.setdefault(name, [])
                parts.append(out[name])
                # circular buffer: drop whole chunks that can no longer contribute to the last `keephistory` ticks
                field = "mu" if hasattr(out[name], "mu") else ("m" if hasattr(out[name], "m") else "a")
                total = sum(getattr(p, field).shape[0] for p in parts)
                while len(parts) > 1 and total - getattr(parts[0], field).shape[0] >= self.keephistory:
                    total -= getattr(parts.pop(0), field).shape[0]

    # -------------------------------------------------------------- results (streaming.jl:16-140)
    @property
    def posteriors(self):
        """Most recent marginals (the reference exposes observables; here: the last tick's values)."""
        if self._kind == "lgssm":
            return {"x_t": (self._prev_mean, self._carry_cov.copy())}
        if self._kind == "delta":            # per-chain carry, [d, batch] / [d, d, batch] (and (shape, rate) [batch])
            q = {("state" if self._tau is not None else "x_t"): MvNormalMeanCovariance(self._mean, self._cov)}
            if self._tau is not None:
                q["noise"] = GammaShapeRate(self._tau[0], self._tau[1])
            return q
        if self._kind == "multinomial":      # fp64 carry, [D, batch] / [D, D, batch]
            return {"ψ": None if self._carry is None else MvNormalMeanCovariance(*self._carry)}
        if self._kind == "vmpgamma":
            c = self._carry
            return {"x_t": None if c is None else NormalMeanVariance(c[0], c[1]),
                    "τ": None if c is None else GammaShapeRate(c[2], c[3])}
        return {"xt": None if self._carry is None else NormalMeanVariance(self._carry[0], self._carry[1]),
                "zt": None if self._carry is None else NormalMeanVariance(self._carry[2], self._carry[3])}

    @property
    def history(self):
        """Last ``keephistory`` marginals per history variable, concatenated along time (circular buffer)."""
        if not self.keephistory:
            raise RuntimeError("history has not been kept: use the `keephistory` argument")   # streaming.jl getproperty
        out = {}
        for name, parts in self._hist.items():
            first = parts[0]
            fields = [f for f in ("mu", "Sigma", "m", "v", "a", "b") if hasattr(first, f)]
            cat = {f: torch.cat([getattr(p, f) for p in parts], dim=0)[-self.keephistory:] for f in fields}
            out[name] = type(first)(**cat)
        return out

    @property
    def free_energy_history(self):
        """Per chunk: -log p(y_chunk | past) per chain, stacked [n_chunks, batch]; their sum over chunks is the
        evidence of the whole stream (on this tree BFE = -log evidence)."""
        if not self.free_energy_enabled:
            raise RuntimeError("Bethe Free Energy has not been computed: use `free_energy = true`")
        if self._kind == "multinomial":
            raise NotImplementedError("the multinomial regression keeps the free energy of each datum's final iteration "
                                      "only: free_energy_final_only_history")
        if self._kind in ("vmpgamma", "hgf"):   # reference semantics (streaming.jl:12): per iteration, averaged over the observations
            return torch.cat(self._fe, dim=0).mean(dim=0)
        return torch.stack(self._fe)

    @property
    def free_energy_final_only_history(self):
        """The free energy of each datum's final iteration, [ticks, batch] (fp64): KL(q_t || q_{t-1}) minus the bound of
        datum t's evidence (multinomial regression)."""
        if not self.free_energy_enabled:
            raise RuntimeError("Bethe Free Energy has not been computed: use `free_energy = true`")
        if self._kind != "multinomial":
            raise NotImplementedError("free_energy_final_only_history is kept by the multinomial regression engine")
        return torch.cat(self._fe, dim=0)
