"""Thin object wrapper over the C ABI: one ``Context`` per GPU / host thread.

PyTorch is used only as plumbing (device memory, the current stream); every computation goes
through ``librxgauss.so``.
"""
from __future__ import annotations

import ctypes
from ctypes import c_void_p
from types import SimpleNamespace

import numpy as np
import torch

from . import _lib as L


def _fp(t):
    if t is None:
        return L.as_fp(0)
    return L.as_fp(t.data_ptr())


def _i32(t):
    return ctypes.cast(c_void_p(t.data_ptr() if t is not None else None), L.i32p)


def _f64(t):
    return ctypes.cast(c_void_p(t.data_ptr() if t is not None else None), ctypes.POINTER(ctypes.c_double))


def _u8(t):
    return ctypes.cast(c_void_p(t.data_ptr() if t is not None else None), L.u8p)


def _model32(M):
    """Shared model matrices are small host arrays (row-major fp32)."""
    a = np.ascontiguousarray(np.asarray(M, dtype=np.float32))
    return a, a.ctypes.data_as(L.fp)


def _host_arrays(who, arrays, dims, nulls=False):
    """The host model arrays of one C entry, shape-checked and packed to row-major fp32: ``arrays`` maps each name to
    (value, expected shape); with ``nulls`` a None value is a null pointer.  ``dims`` names the sizes in the error text
    (``"K = 3, d = 2"``).  Returns {name: (array, pointer)}; the arrays must outlive the call."""
    keep = {}
    for k, (v, shp) in arrays.items():
        if v is None and nulls:
            keep[k] = (None, L.as_fp(0))
            continue
        keep[k] = _model32(v)
        if keep[k][0].shape != shp:
            raise ValueError(f"{who}: {k}: expected shape {shp} ({dims}), got {keep[k][0].shape}")
    return keep


def delta_mask(mask, T, batch, device, who):
    """The Delta kernels read ymask[t][b] for every step and chain: a mask must be [T, batch] exactly (checked on the
    host, before anything is copied or launched).  Returns it as contiguous uint8 on ``device``, or None."""
    if mask is None:
        return None
    shape = tuple(mask.shape) if hasattr(mask, "shape") else tuple(np.shape(mask))
    if shape != (T, batch):
        raise ValueError(f"{who}: mask must be [T, batch] = {(T, batch)} (1 = observed), got {shape}")
    return torch.as_tensor(mask, device=device).to(torch.uint8).contiguous()


class Context:
    """``rxg_ctx`` bound to a CUDA device.  Launches go to torch's current stream on that device
    (so ``torch.cuda.Event`` timing and stream ordering with torch ops are meaningful)."""

    def __init__(self, device: int | None = None, use_torch_stream: bool = True):
        self.lib = L.load()
        if not torch.cuda.is_available():
            raise L.RxGaussError(L.RXG_ERR_NO_DEVICE, "no CUDA device: the hot path has no CPU fallback")
        self.device = torch.cuda.current_device() if device is None else int(device)
        h = c_void_p()
        rc = self.lib.rxg_create(ctypes.byref(h), self.device, 0)
        if rc != 0:
            raise L.RxGaussError(rc, "rxg_create failed")
        self.h = h
        self._stream = None
        if use_torch_stream:
            self.bind_stream()

    # ------------------------------------------------------------------ plumbing
    def bind_stream(self, stream: torch.cuda.Stream | None = None):
        s = stream if stream is not None else torch.cuda.current_stream(self.device)
        self._stream = s
        self._check(self.lib.rxg_set_stream(self.h, c_void_p(s.cuda_stream)))

    def _check(self, rc):
        if rc != 0:
            raise L.RxGaussError(rc, self.lib.rxg_last_error(self.h).decode())

    def sync(self):
        self._check(self.lib.rxg_sync(self.h))

    @property
    def launches(self) -> int:
        return int(self.lib.rxg_launch_count(self.h))

    def host_fill_threads(self) -> int:
        return int(self.lib.rxg_host_fill_threads())

    OPTIONS = {"gain_seq": 0, "large_seq": 1, "no_umma": 2, "sweep_variant": 3, "force_cpt": 4, "host_threads": 5,
               "host_cov_d2h": 6, "host_bcast_min_mb": 7, "host_slices": 8, "gather_mode": 9, "polya_path": 10}

    def set_option(self, name: str, value: int):
        """``rxg_set_option``: per-context dispatch switches (cross-check kernels, host-pipeline tuning)."""
        self._check(self.lib.rxg_set_option(self.h, self.OPTIONS[name], int(value)))

    def get_option(self, name: str) -> int:
        v = ctypes.c_longlong()
        self._check(self.lib.rxg_get_option(self.h, self.OPTIONS[name], ctypes.byref(v)))
        return int(v.value)

    def set_profiling(self, on=True):
        self._check(self.lib.rxg_set_profiling(self.h, 1 if on else 0))

    def profile_last_ms(self):
        a, b = ctypes.c_float(), ctypes.c_float()
        self._check(self.lib.rxg_profile_last_ms(self.h, ctypes.byref(a), ctypes.byref(b)))
        return a.value, b.value

    def close(self):
        if getattr(self, "h", None):
            self.lib.rxg_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _dev(self, *ts):
        for t in ts:
            if t is None:
                continue
            if not (t.is_cuda and t.dtype == torch.float32 and t.is_contiguous()):
                raise ValueError("expected contiguous float32 CUDA tensors")
            if t.device.index != self.device:
                raise ValueError(f"tensor lives on cuda:{t.device.index}, this context is bound to cuda:{self.device}")

    def _io(self, t, name, on_dev=True, dtype=torch.float32, shape=None, ndim=None):
        """Validate one tensor an entry reads or writes (None passes): dtype, contiguity, on this context's device (or
        on the host), then its shape or its number of dimensions.  Dtype, contiguity and host / device come first, so
        that they are checked without ``self.device``."""
        if t is None:
            return
        if not isinstance(t, torch.Tensor) or t.dtype != dtype or not t.is_contiguous():
            got = f"{t.dtype}, contiguous={t.is_contiguous()}" if isinstance(t, torch.Tensor) else type(t).__name__
            raise ValueError(f"{name}: expected a contiguous {dtype} tensor, got {got} (call .contiguous() / "
                             f".to({dtype}) explicitly)")
        if on_dev and not t.is_cuda:
            raise ValueError(f"{name}: expected a tensor on cuda (y is a device array), got {t.device}")
        if on_dev and t.device.index != self.device:
            raise ValueError(f"{name}: expected a tensor on cuda:{self.device} (y is a device array), got {t.device}")
        if not on_dev and t.is_cuda:
            raise ValueError(f"{name}: y is a host array, so every data array must be on the host; got {t.device}")
        if shape is not None and tuple(t.shape) != tuple(shape):
            raise ValueError(f"{name}: expected shape {tuple(shape)}, got {tuple(t.shape)}")
        if ndim is not None and t.dim() != ndim:
            raise ValueError(f"{name}: expected {ndim} dimensions, got shape {tuple(t.shape)}")

    def empty(self, *shape, dtype=torch.float32):
        return torch.empty(*shape, dtype=dtype, device=f"cuda:{self.device}")

    # ------------------------------------------------------------------ fused sweeps
    def _inputs(self, inputs, u, rows, d, batch):
        """Known per-step inputs (``inputs=``): a CPU / numpy [rows, d] array is one sequence for every chain
        (RXG_U_SEQ_SHARED), a CUDA [rows, d, batch] tensor one per chain (RXG_U_SEQ_CHAIN).  Row t enters the transition
        into x[t].  Returns (flag, pointer, kept array) or None."""
        if inputs is None:
            return None
        if u is not None:
            raise ValueError("pass either a constant offset u or an input sequence inputs, not both "
                             "(fold the constant into the sequence)")
        if isinstance(inputs, torch.Tensor) and inputs.is_cuda:
            self._io(inputs, "inputs", True, shape=(rows, d, batch))
            return L.U_SEQ_CHAIN, _fp(inputs), inputs
        a = np.ascontiguousarray(np.asarray(inputs.cpu() if isinstance(inputs, torch.Tensor) else inputs, dtype=np.float32))
        if a.shape != (rows, d):
            raise ValueError(f"inputs: expected a host array of shape {(rows, d)} (or a CUDA tensor {(rows, d, batch)}), "
                             f"got {a.shape}")
        return L.U_SEQ_SHARED, a.ctypes.data_as(L.fp), a

    def _sweep_args(self, y, A, B, P, Q, m0, S0, u, mask, on_dev, per_chain_model, force_per_chain_path, cov_shared_out,
                    transition_first, asynchronous, inputs=None, input_rows=None):
        """Validation, flags and pointers shared by the fused LGSSM sweeps: returns (T, m, batch, d, flags, ptrs, mask,
        mask_p, keep) -- ``mask`` the per-chain mask tensor or None, ``keep`` the host arrays that must outlive the call."""
        if y.dim() != 3:
            raise ValueError(f"y: expected [T, m, batch], got shape {tuple(y.shape)}")
        T, m, batch = y.shape
        self._io(y, "y", on_dev)
        shared_mask = None
        if mask is not None and getattr(mask, "ndim", 2) == 1:
            # one missing-data pattern for every chain (RXG_MASK_SHARED): a host array [T]; the call stays on the gain-table path
            shared_mask = np.ascontiguousarray(np.asarray(mask.cpu() if isinstance(mask, torch.Tensor) else mask, dtype=np.uint8))
            if shared_mask.shape != (T,):
                raise ValueError(f"shared mask: expected shape ({T},), got {shared_mask.shape}")
            mask = None
        self._io(mask, "mask", on_dev, dtype=torch.uint8, shape=(T, batch))
        flags = L.PTR_DEVICE if on_dev else 0
        if shared_mask is not None:
            flags |= L.MASK_SHARED
        if per_chain_model:
            flags |= L.MODEL_PER_CHAIN
            d = A.shape[0]
            self._dev(A, B, P, Q, m0, S0, u)
            ptrs = [_fp(x) for x in (A, B, P, Q, m0, S0, u)]
            keep = []
        else:
            d = np.asarray(A).shape[-1]
            keep = [_model32(x) for x in (A, B, P, Q, m0, S0)]
            ptrs = [k[1] for k in keep]
            if u is not None:
                keep.append(_model32(u))
                ptrs.append(keep[-1][1])
            else:
                ptrs.append(L.as_fp(0))
        if force_per_chain_path:
            flags |= L.PATH_PER_CHAIN
        if cov_shared_out:
            flags |= L.COV_SHARED_OUT
        if transition_first:
            flags |= L.TRANSITION_FIRST
        if asynchronous:
            flags |= L.ASYNC
        seq = self._inputs(inputs, u, T if input_rows is None else input_rows, d, batch)
        if seq is not None:
            flags |= seq[0]
            ptrs[-1] = seq[1]
            keep.append(seq[2])
        mask_p = ctypes.cast(c_void_p(mask.data_ptr()), L.u8p) if mask is not None else ctypes.cast(c_void_p(None), L.u8p)
        if shared_mask is not None:
            mask_p = shared_mask.ctypes.data_as(L.u8p)
            keep.append(shared_mask)
        return T, m, batch, d, flags, ptrs, mask, mask_p, keep

    def lgssm(self, y, A, B, P, Q, m0, S0, *, u=None, inputs=None, smooth=True, mask=None, want_cov=True,
              want_evidence=False, want_status=False, per_chain_model=False, force_per_chain_path=False, cov_shared_out=False,
              transition_first=False, out_mean=None, out_cov=None, out_status=None, asynchronous=False):
        """y[T, m, batch] (CUDA fp32, or pinned/pageable CPU fp32 for the host-pointer path)
        -> dict(mean[T,d,batch], cov[T,d,d,batch] or [T,d,d], neg_log_evidence[batch], status[batch]).
        ``inputs``: known per-step inputs, x[t] ~ N(A x[t-1] + inputs[t], P) -- a host [T, d] array shared by every
        chain, or a CUDA [T, d, batch] tensor (device calls only); exclusive with ``u``."""
        on_dev = y.is_cuda
        T, m, batch, d, flags, ptrs, mask, mask_p, keep = self._sweep_args(
            y, A, B, P, Q, m0, S0, u, mask, on_dev, per_chain_model, force_per_chain_path, cov_shared_out, transition_first,
            asynchronous, inputs)
        mk = lambda *s, dt=torch.float32: (torch.empty(*s, dtype=dt, device=y.device) if on_dev
                                           else torch.empty(*s, dtype=dt).pin_memory())
        self._io(out_mean, "out_mean", on_dev, shape=(T, d, batch))
        self._io(out_cov, "out_cov", on_dev, shape=(T, d, d) if cov_shared_out else (T, d, d, batch))
        mean = out_mean if out_mean is not None else mk(T, d, batch)
        need_cov = want_cov or per_chain_model or force_per_chain_path or mask is not None
        cov = out_cov
        if cov is None and need_cov:
            cov = mk(T, d, d) if cov_shared_out else mk(T, d, d, batch)
        nle = mk(batch) if want_evidence else None
        self._io(out_status, "out_status", on_dev, dtype=torch.int32, shape=(batch,))
        status = out_status if out_status is not None else (mk(batch, dt=torch.int32) if want_status else None)
        fn = self.lib.rxg_lgssm_smooth_f32 if smooth else self.lib.rxg_lgssm_filter_f32
        st_p = ctypes.cast(c_void_p(status.data_ptr()), L.i32p) if status is not None else ctypes.cast(c_void_p(None), L.i32p)
        self._check(fn(self.h, d, m, T, batch, *ptrs, _fp(y), mask_p, _fp(mean), _fp(cov), _fp(nle), st_p, flags))
        return dict(mean=mean, cov=cov if (want_cov or need_cov) else None, neg_log_evidence=nle, status=status)

    def lgssm_predict(self, y, A, B, P, Q, m0, S0, *, horizon=0, u=None, inputs=None, mask=None, want_cov=True, want_pred_cov=True,
                      want_forecast_states=True, want_evidence=False, want_status=False, per_chain_model=False,
                      force_per_chain_path=False, cov_shared_out=False, transition_first=False, asynchronous=False):
        """Smoother + predictive distributions of the observations (``rxg_lgssm_smooth_predict_f32``).
        y[T, m, batch] on this context's device; ``mask`` as for :meth:`lgssm` ([T, batch] per chain, or a [T] pattern
        shared by every chain).  Returns dict(mean, cov, neg_log_evidence, status) as :meth:`lgssm` plus
        pred_mean[T+H, m, batch], pred_cov[T+H, m, m, batch] (or [T+H, m, m] with ``cov_shared_out``), and the state
        forecasts fc_mean[H, d, batch], fc_cov[H, d, d, batch] (or [H, d, d]); rows T.. of pred_* are the forecasts.
        ``inputs`` as for :meth:`lgssm` with T + H rows: forecast k = 1..H uses row T + k - 1."""
        if not y.is_cuda:
            raise ValueError("lgssm_predict: y must be a CUDA tensor (the prediction entry takes device pointers)")
        H = int(horizon)
        if H < 0:
            raise ValueError(f"horizon must be >= 0, got {horizon}")
        T, m, batch, d, flags, ptrs, mask, mask_p, keep = self._sweep_args(
            y, A, B, P, Q, m0, S0, u, mask, True, per_chain_model, force_per_chain_path, cov_shared_out, transition_first,
            asynchronous, inputs, y.shape[0] + H)
        mk = lambda *s, dt=torch.float32: torch.empty(*s, dtype=dt, device=y.device)
        mean = mk(T, d, batch)
        need_cov = want_cov or per_chain_model or force_per_chain_path or mask is not None
        cov = (mk(T, d, d) if cov_shared_out else mk(T, d, d, batch)) if need_cov else None
        nle = mk(batch) if want_evidence else None
        status = mk(batch, dt=torch.int32) if want_status else None
        pred_mean = mk(T + H, m, batch)
        pred_cov = (mk(T + H, m, m) if cov_shared_out else mk(T + H, m, m, batch)) if want_pred_cov else None
        fc_mean = mk(H, d, batch) if (H > 0 and want_forecast_states) else None
        fc_cov = (mk(H, d, d) if cov_shared_out else mk(H, d, d, batch)) if (H > 0 and want_forecast_states) else None
        st_p = ctypes.cast(c_void_p(status.data_ptr()), L.i32p) if status is not None else ctypes.cast(c_void_p(None), L.i32p)
        self._check(self.lib.rxg_lgssm_smooth_predict_f32(self.h, d, m, T, H, batch, *ptrs, _fp(y), mask_p, _fp(mean), _fp(cov),
                                                          _fp(nle), _fp(pred_mean), _fp(pred_cov), _fp(fc_mean), _fp(fc_cov),
                                                          st_p, flags))
        return dict(mean=mean, cov=cov if want_cov else None, neg_log_evidence=nle, status=status, pred_mean=pred_mean,
                    pred_cov=pred_cov, fc_mean=fc_mean, fc_cov=fc_cov)

    def lgssm_filter_chunk(self, y, A, B, P, Q, prev_mean, carry_cov, *, u=None, inputs=None, want_evidence=False,
                           cov_shared_out=False, out_mean=None, out_cov=None):
        """One time-chunk of the streaming engine (``rxg_lgssm_filter_chunk_f32``).  ``prev_mean[d, batch]``
        (CUDA) and ``carry_cov[d, d]`` (host fp32 numpy, updated IN PLACE) are the autoupdate carry.  ``inputs``: the
        chunk's input rows ([Tc, d] host or [Tc, d, batch] CUDA, as for :meth:`lgssm`; row 0 enters x[t0])."""
        self._dev(y, prev_mean)
        T, m, batch = y.shape
        d = prev_mean.shape[0]
        if not (isinstance(carry_cov, np.ndarray) and carry_cov.dtype == np.float32 and carry_cov.shape == (d, d)
                and carry_cov.flags.c_contiguous):
            raise ValueError("carry_cov must be a C-contiguous float32 numpy array of shape (d, d)")
        keep = [_model32(x) for x in (A, B, P, Q)]
        ptrs = [k[1] for k in keep]
        if u is not None:
            keep.append(_model32(u))
            ptrs.append(keep[-1][1])
        else:
            ptrs.append(L.as_fp(0))
        mean = out_mean if out_mean is not None else self.empty(T, d, batch)
        cov = out_cov if out_cov is not None else (self.empty(T, d, d) if cov_shared_out else self.empty(T, d, d, batch))
        nle = self.empty(batch) if want_evidence else None
        flags = L.PTR_DEVICE | (L.COV_SHARED_OUT if cov_shared_out else 0)
        seq = self._inputs(inputs, u, T, d, batch)
        if seq is not None:
            flags |= seq[0]
            ptrs[-1] = seq[1]
            keep.append(seq[2])
        cc = carry_cov.ctypes.data_as(L.fp)
        self._check(self.lib.rxg_lgssm_filter_chunk_f32(self.h, d, m, T, batch, *ptrs, _fp(prev_mean), cc, _fp(y),
                                                        _fp(mean), _fp(cov), _fp(nle), flags))
        return dict(mean=mean, cov=cov, neg_log_evidence=nle)

    # ------------------------------------------------------------------ Delta node (user functions, NVRTC)
    def delta_model(self, source, f_name, d, m, method, g_name=None, ut=None):
        """``rxg_delta_model_create``: compile (or find in this context's cache) the module of the user functions
        ``f_name`` (R^d -> R^d) and ``g_name`` (R^d -> R^m, or None) defined in the CUDA ``source``; ``method`` is
        ``L.RXG_DELTA_LINEARIZATION`` or ``L.RXG_DELTA_UNSCENTED`` with ``ut = (alpha, beta, kappa)`` or None for the
        defaults.  A compile error raises ``RxGaussError`` carrying the NVRTC log."""
        log = ctypes.create_string_buffer(1 << 16)
        h = c_void_p()
        uta = (ctypes.c_double * 3)(*ut) if ut is not None else None
        rc = self.lib.rxg_delta_model_create(self.h, source.encode(), f_name.encode(), g_name.encode() if g_name else None,
                                             int(d), int(m), int(method), uta, ctypes.byref(h), log, len(log))
        self._check(rc)
        return SimpleNamespace(h=h, d=int(d), m=int(m), method=int(method), has_g=g_name is not None)

    @property
    def delta_compiles(self) -> int:
        """NVRTC compilations this context has run (a cached ``delta_model`` adds none)."""
        return int(self.lib.rxg_delta_compile_count(self.h))

    def _delta_consts(self, model, **arrays):
        d, m = model.d, model.m
        shapes = {"m0": (d,), "S0": (d, d), "P": (d, d), "B": (m, d), "Q": (m, m)}
        return _host_arrays("delta", {k: (v, shapes[k]) for k, v in arrays.items()}, f"d = {d}, m = {m}", nulls=True)

    def delta_smooth(self, model, y, m0, S0, P, Q, B=None, mask=None, want_filtered=False):
        """``rxg_delta_smooth_f32``: y[T, m, batch] (CUDA fp32), mask[T, batch] (uint8 / bool) or None.  Returns mean
        [T, d, batch], cov [T, d, d, batch], status [batch] and, with ``want_filtered``, filt_mean / filt_cov."""
        self._io(y, "delta_smooth: y [T, m, batch]", ndim=3)
        T, m, batch = y.shape
        if m != model.m:
            raise ValueError(f"delta_smooth: y has m = {m}, the model m = {model.m}")
        d = model.d
        k = self._delta_consts(model, m0=m0, S0=S0, P=P, B=B, Q=Q)
        mk = delta_mask(mask, T, batch, y.device, "delta_smooth")
        mean, cov = self.empty(T, d, batch), self.empty(T, d, d, batch)
        fm = self.empty(T, d, batch) if want_filtered else None
        fc = self.empty(T, d, d, batch) if want_filtered else None
        st = self.empty(batch, dtype=torch.int32)
        self._check(self.lib.rxg_delta_smooth_f32(self.h, model.h, T, batch, k["m0"][1], k["S0"][1], k["P"][1], k["B"][1],
                                                  k["Q"][1], _fp(y), _u8(mk), _fp(mean), _fp(cov), _fp(fm), _fp(fc),
                                                  _i32(st), L.PTR_DEVICE))
        return dict(mean=mean, cov=cov, filt_mean=fm, filt_cov=fc, status=st)

    def delta_filter_chunk(self, model, y, P, carry_mean, carry_cov, Q=None, B=None, carry_tau=None, iters=1, mask=None,
                           want_history=True):
        """``rxg_delta_filter_chunk_f32``: one time-chunk y[Tc, m, batch] of the streaming filter.  The carry
        ``carry_mean[d, batch]`` / ``carry_cov[d, d, batch]`` (and ``carry_tau[2, batch]`` = (shape, rate) of a learned
        precision, m = 1, ``B`` the observation row, no ``Q``) are CUDA fp32 tensors updated in place.  Returns the
        chunk's filtered mean / cov (and tau [Tc, 2, batch]) when ``want_history``, and status [batch]."""
        self._io(y, "delta_filter_chunk: y [Tc, m, batch]", ndim=3)
        T, m, batch = y.shape
        if m != model.m:
            raise ValueError(f"delta_filter_chunk: y has m = {m}, the model m = {model.m}")
        d = model.d
        for t, name, shp in ((carry_mean, "carry_mean", (d, batch)), (carry_cov, "carry_cov", (d, d, batch)),
                             (carry_tau, "carry_tau", (2, batch))):
            self._io(t, f"delta_filter_chunk: {name}", shape=shp)
        k = self._delta_consts(model, P=P, B=B, Q=Q)
        mk = delta_mask(mask, T, batch, y.device, "delta_filter_chunk")
        fm = self.empty(T, d, batch) if want_history else None
        fc = self.empty(T, d, d, batch) if want_history else None
        ft = self.empty(T, 2, batch) if want_history and carry_tau is not None else None
        st = self.empty(batch, dtype=torch.int32)
        self._check(self.lib.rxg_delta_filter_chunk_f32(self.h, model.h, T, batch, k["P"][1], k["B"][1], k["Q"][1],
                                                        int(iters), _fp(y), _u8(mk), _fp(carry_mean), _fp(carry_cov),
                                                        _fp(carry_tau), _fp(fm), _fp(fc), _fp(ft), _i32(st),
                                                        L.PTR_DEVICE))
        return dict(mean=fm, cov=fc, tau=ft, status=st)

    HGF_LEARN_PRIOR = (1.0, 1.0, 0.0, 1.0, 0.0, 1.0, 0.0, 1.0)   # hgf_1: kappa, omega, x_0, z[1] ~ N(mean, variance)
    HGF_LEARN_INIT = (1.0, 1.0, 0.0, 1.0, 0.0, 1.0, 0.0, 1.0)    # initial q(kappa), q(omega), q(z), q(x)

    def hgf_vmp_learn(self, y, prior=HGF_LEARN_PRIOR, z_precision=1.0, y_variance=1.0, init=HGF_LEARN_INIT, iterations=1,
                      want_free_energy=True, keep_each=False):
        """``rxg_hgf_vmp_learn_f32``: mean-field VMP of the HGF with kappa and omega learned per series.  y[T, batch] fp32
        on the device (NaN = missing step); ``prior`` = (mean, variance) of kappa, omega, x_0, z[1]; ``init`` = (mean,
        variance) of the initial q(kappa), q(omega), q(z[t]), q(x[t]).  Returns ``xz[T, 4, batch]`` = (m_x, v_x, m_z, v_z),
        ``x0[2, batch]``, ``kw[2, 2, batch]`` = (mean, variance) of q(kappa) then q(omega), ``free_energy[iterations,
        batch]`` (fp64) or None, ``status[batch]`` and, with ``keep_each``, ``hist_kw[iterations, 2, 2, batch]``."""
        self._io(y, "hgf_vmp_learn: y [T, batch]", ndim=2)
        T, batch = y.shape
        pr, ini = np.asarray(prior, np.float32).reshape(-1), np.asarray(init, np.float32).reshape(-1)
        if pr.shape != (8,) or ini.shape != (8,):
            raise ValueError("hgf_vmp_learn: prior and init are 8 numbers each ((mean, variance) of four variables)")
        its = int(iterations)
        xz, x0, kw = self.empty(T, 4, batch), self.empty(2, batch), self.empty(2, 2, batch)
        hist = self.empty(its, 2, 2, batch) if keep_each else None
        fe = self.empty(its, batch, dtype=torch.float64) if want_free_energy else None
        st = self.empty(batch, dtype=torch.int32)
        self._check(self.lib.rxg_hgf_vmp_learn_f32(self.h, T, batch, its, pr.ctypes.data_as(L.fp), float(z_precision),
                                                   float(y_variance), ini.ctypes.data_as(L.fp), _fp(y), _fp(x0), _fp(xz),
                                                   _fp(kw), _fp(hist), _f64(fe), _i32(st), L.PTR_DEVICE))
        return dict(xz=xz, x0=x0, kw=kw, hist_kw=hist, free_energy=fe, status=st)

    def hgf_filter_chunk(self, y, prev, iters=20, kappa=1.0, omega=0.0, z_variance=0.04, y_variance=0.01, out=None,
                         want_free_energy=False):
        """HGF datastream chunk; ``prev[4, batch]`` = ``out[-1]`` of the previous chunk."""
        return self.hgf_filter(y, iters, kappa, omega, z_variance, y_variance, init=None, out=out, prev=prev,
                               want_free_energy=want_free_energy)

    def hgf_filter(self, y, iters=20, kappa=1.0, omega=0.0, z_variance=0.04, y_variance=0.01,
                   init=(0.0, 5.0, 0.0, 5.0), out=None, prev=None, want_free_energy=False):
        """``rxg_hgf_filter_fe_f32``: y[T, batch] -> out[T, 4, batch] = (m_x, v_x, m_z, v_z); with
        ``want_free_energy`` also the Bethe free energy [T, iters, batch] (returned as a pair)."""
        self._dev(y, prev, out)
        T, batch = y.shape
        out = out if out is not None else self.empty(T, 4, batch)
        fe = self.empty(T, iters, batch) if want_free_energy else None
        ini = ctypes.cast((ctypes.c_float * 4)(*init), L.fp) if prev is None else L.as_fp(0)
        self._check(self.lib.rxg_hgf_filter_fe_f32(self.h, T, batch, iters, kappa, omega, z_variance, y_variance,
                                                   ini, _fp(prev), _fp(y), _fp(out), _fp(fe), L.PTR_DEVICE))
        return (out, fe) if want_free_energy else out

    def stream_vmp_gamma(self, y, iters=4, w=1.0, init=(0.0, 1e3, 1.0, 1.0), prev=None, want_free_energy=False):
        """Streaming mean-field VMP with a Gamma observation precision (``rxg_stream_vmp_gamma_f32``);
        y[T, batch] -> out[T, 4, batch] = (m_x, v_x, shape, rate), free energy [T, iters, batch] or None."""
        self._dev(y, prev)
        T, batch = y.shape
        out = self.empty(T, 4, batch)
        fe = self.empty(T, iters, batch) if want_free_energy else None
        ini = (ctypes.c_float * 4)(*init)
        self._check(self.lib.rxg_stream_vmp_gamma_f32(self.h, T, batch, iters, w, ctypes.cast(ini, L.fp), _fp(prev), _fp(y),
                                                      _fp(out), _fp(fe), L.PTR_DEVICE))
        return out, fe

    def lgssm_vmp_gamma(self, y, iterations=10, a=1.0, v_proc=1.0, prior=(0.0, 100.0), gamma_prior=(1.0, 1.0),
                        init_E_tau=1.0, want_free_energy=False):
        self._dev(y)
        T, batch = y.shape
        pm, pv = self.empty(T, batch), self.empty(T, batch)
        sh, rt = self.empty(batch), self.empty(batch)
        fe = self.empty(iterations, batch) if want_free_energy else None
        self._check(self.lib.rxg_lgssm_vmp_gamma_fe_f32(self.h, T, batch, iterations, a, v_proc, prior[0], prior[1],
                                                        gamma_prior[0], gamma_prior[1], init_E_tau, _fp(y), _fp(pm),
                                                        _fp(pv), _fp(sh), _fp(rt), _fp(fe), L.PTR_DEVICE))
        return dict(mean=pm, var=pv, shape=sh, rate=rt, free_energy=fe)

    def lgssm_vmp_wishart(self, y, A, B, P, m0, S0, iterations=10, w_prior=None, init_E_W=None, u=None, mask=None,
                          transition_first=False, want_free_energy=False, asynchronous=False):
        """VMP around the smoother with an unknown observation precision matrix per chain (``rxg_lgssm_vmp_wishart_f32``):
        w ~ Wishart(nu0, inv(inv_scale0)), x[t] ~ N(A x[t-1] + u, P), y[t] ~ N(B x[t], inv(w)), q(x) q(w).
        y[T, m, batch] on this context's device; ``mask`` as for :meth:`lgssm` ([T, batch] per chain or a [T] pattern
        shared by every chain).  ``w_prior = (nu0, inv_scale0)`` (default (m + 1, I)); ``init_E_W`` = E[w] of the
        initial q(w) (default: the mean of ``vague(Wishart, m)``, m * 1e12 I).  Returns dict(mean[T, d, batch],
        cov[T, d, d, batch] of the last iteration, df[iterations, batch], inv_scale[iterations, m, m, batch] after every
        iteration, free_energy[iterations, batch] fp64 or None, status[batch])."""
        m = self._vmp_dims(y)[1]
        d = np.asarray(A).shape[-1]
        if w_prior is None:
            w_prior = (m + 1.0, np.eye(m))
        if init_E_W is None:
            init_E_W = m * 1e12 * np.eye(m)                     # mean of vague(Wishart, m): df = m, scale 1e12 I
        c = self._vmp_setup("lgssm_vmp_wishart", y, d, dict(A=A), dict(A=(d, d)), B, m0, S0, P, None, None, None,
                            w_prior, init_E_W, u, iterations, mask, transition_first, asynchronous, want_free_energy,
                            q_keys=("inv_scale0", "init_E_W"))
        self._check(self.lib.rxg_lgssm_vmp_wishart_f32(       # this entry has no known Q and no outputs for P
            *c.head, c.hp("A"), c.hp("B"), c.hp("P"), c.hp("m0"), c.hp("S0"), c.hp("u"), *c.q[1:], *c.io, *c.w_out[2:],
            *c.tail))
        return dict(mean=c.mean, cov=c.cov, df=c.out["df_q"], inv_scale=c.out["inv_scale_q"], free_energy=c.fe,
                    status=c.st)

    def _vmp_mask_flags(self, mask, T, batch, keep, transition_first, asynchronous):
        """Mask pointer and flags of the Wishart VMP entries: a [T, batch] device mask per chain or a [T] pattern shared by
        every chain (staged from the host; kept alive in ``keep``)."""
        flags = L.PTR_DEVICE
        mask_p = _u8(None)
        if mask is not None and getattr(mask, "ndim", 2) == 1:
            sm = np.ascontiguousarray(np.asarray(mask.cpu() if isinstance(mask, torch.Tensor) else mask, dtype=np.uint8))
            if sm.shape != (T,):
                raise ValueError(f"shared mask: expected shape ({T},), got {sm.shape}")
            keep["mask"] = sm
            mask_p = sm.ctypes.data_as(L.u8p)
            flags |= L.MASK_SHARED
        elif mask is not None:
            self._io(mask, "mask", True, dtype=torch.uint8, shape=(T, batch))
            mask_p = _u8(mask)
        if transition_first:
            flags |= L.TRANSITION_FIRST
        if asynchronous:
            flags |= L.ASYNC
        return mask_p, flags

    def lgssm_vmp_noise(self, y, A, B, m0, S0, *, P=None, Q=None, p_prior=None, p_init=None, q_prior=None, q_init=None,
                        u=None, mask=None, transition_first=False, iterations=10, want_free_energy=False,
                        asynchronous=False):
        """VMP around the smoother with an unknown process precision matrix w_p, alone or together with an unknown
        observation precision w_q, one of each per chain (``rxg_lgssm_vmp_noise_f32``):
        w_p ~ Wishart(nu_p0, inv(inv_scale_p0)), w_q ~ Wishart(nu_q0, inv(inv_scale_q0)), x[t] ~ N(A x[t-1] + u, inv(w_p)),
        y[t] ~ N(B x[t], inv(w_q)), q(x) q(w_p) q(w_q).  For each noise pass either the known matrix (``P`` / ``Q``) or the
        prior ``(nu0, inv_scale0)`` together with ``*_init`` = E[w] of the initial q(w); a learned noise has no default
        initial q(w) (a vague one makes the first fp32 sweep ill-conditioned).  y[T, m, batch] on this context's device;
        ``mask`` as for :meth:`lgssm_vmp_wishart`.  Returns dict(mean[T, d, batch], cov[T, d, d, batch] of the last
        iteration, df_p[iterations, batch] / inv_scale_p[iterations, d, d, batch] and df_q / inv_scale_q ([.., m, m, ..])
        after every iteration (None for a known noise), free_energy[iterations, batch] fp64 or None, status[batch])."""
        self._vmp_dims(y)
        d = np.asarray(A).shape[-1]
        c = self._vmp_setup("lgssm_vmp_noise", y, d, dict(A=A), dict(A=(d, d)), B, m0, S0, P, p_prior, p_init, Q,
                            q_prior, q_init, u, iterations, mask, transition_first, asynchronous, want_free_energy,
                            both_known_ok=False)
        self._check(self.lib.rxg_lgssm_vmp_noise_f32(
            *c.head, c.hp("A"), c.hp("B"), c.hp("m0"), c.hp("S0"), c.hp("u"), *c.p, *c.q, *c.io, *c.w_out, *c.tail))
        return dict(mean=c.mean, cov=c.cov, **c.out, free_energy=c.fe, status=c.st)

    @staticmethod
    def _vmp_dims(y):
        if y.dim() != 3:
            raise ValueError(f"y: expected [T, m, batch], got shape {tuple(y.shape)}")
        return y.shape

    def _vmp_setup(self, who, y, d, mats, shapes, B, m0, S0, P, p_prior, p_init, Q, q_prior, q_init, u, iterations,
                   mask, transition_first, asynchronous, want_free_energy, both_known_ok=True,
                   q_keys=("inv_scale_q0", "init_E_Wq")):
        """Shared argument handling of the Wishart VMP entries (``who`` in the error texts): each noise known or
        (prior, init), its host arrays named ``inv_scale_p0`` / ``init_E_Wp`` and ``q_keys`` in the error texts; host
        model arrays converted to row-major fp32 and shape-checked (kept alive in ``keep``); then y and the mask
        validated and the outputs allocated.  Returns the
        pieces of the C call: ``head`` (context and sizes), ``hp(key)`` (a host array's pointer, null if absent), ``p`` /
        ``q`` (known, nu0, inv_scale0, init_E_W), ``io`` (y, mask, mean, cov), ``w_out`` (df_p, inv_scale_p, df_q,
        inv_scale_q; null for a known noise), ``tail`` (free energy, status, flags), next to the output tensors."""
        T, m, batch = y.shape
        iterations = int(iterations)
        if iterations < 1:
            raise ValueError(f"iterations must be >= 1, got {iterations}")
        shapes = dict(shapes, B=(m, d), m0=(d,), S0=(d, d))
        mats = dict(mats, B=B, m0=m0, S0=S0)
        keys = dict(p=("inv_scale_p0", "init_E_Wp"), q=q_keys)
        nus = {}
        for name, k, known, prior, init in (("p", d, P, p_prior, p_init), ("q", m, Q, q_prior, q_init)):
            if known is not None:
                if prior is not None or init is not None:
                    raise ValueError(f"{name.upper()} is known: pass either {name.upper()} or {name}_prior / {name}_init")
                shapes[name.upper()], mats[name.upper()] = (k, k), known
                continue
            if prior is None or init is None:
                raise ValueError(f"{name.upper()} is learned: pass {name}_prior = (nu0, inv_scale0) and {name}_init = E[w] "
                                 f"of the initial q(w_{name}) (there is no default initial q(w))")
            nus[name] = float(prior[0])
            for key, v in zip(keys[name], (prior[1], init)):
                shapes[key], mats[key] = (k, k), v
        if not nus and not both_known_ok:
            raise ValueError("P and Q are both known: that is the plain smoother (Context.lgssm)")
        if u is not None:
            shapes["u"], mats["u"] = (d,), u
        keep = _host_arrays(who, {k: (v, shapes[k]) for k, v in mats.items()}, f"d = {d}, m = {m}")
        self._io(y, "y", True)
        mask_p, flags = self._vmp_mask_flags(mask, T, batch, keep, transition_first, asynchronous)
        c = SimpleNamespace(keep=keep, iterations=iterations, batch=batch, mean=self.empty(T, d, batch),
                            cov=self.empty(T, d, d, batch), out={})
        for name, k in (("p", d), ("q", m)):
            learned = name in nus
            c.out[f"df_{name}"] = self.empty(iterations, batch) if learned else None
            c.out[f"inv_scale_{name}"] = self.empty(iterations, k, k, batch) if learned else None
        c.fe = self.empty(iterations, batch, dtype=torch.float64) if want_free_energy else None
        c.st = self.empty(batch, dtype=torch.int32)
        c.hp = lambda k: keep[k][1] if k in keep else L.as_fp(0)
        c.head = (self.h, d, m, T, batch, iterations)
        c.p, c.q = ((c.hp(name.upper()), nus.get(name, 0.0), *map(c.hp, keys[name])) for name in ("p", "q"))
        c.io = (_fp(y), mask_p, _fp(c.mean), _fp(c.cov))
        c.w_out = tuple(_fp(c.out[k]) for k in ("df_p", "inv_scale_p", "df_q", "inv_scale_q"))
        c.tail = (_f64(c.fe), _i32(c.st), flags)
        return c

    def lgssm_vmp_transition(self, y, B, m0, S0, *, a_prior, a_init, P=None, Q=None, p_prior=None, p_init=None,
                             q_prior=None, q_init=None, u=None, mask=None, transition_first=False, iterations=10,
                             want_free_energy=False, asynchronous=False):
        """VMP around the smoother that also learns the transition matrix A per chain (``rxg_lgssm_vmp_transition_f32``,
        RxInfer's ContinuousTransition with a linear reshape): a = vec(A) ~ N(ma0, Va0), x[t] ~ N(A x[t-1] + u, inv(w_p)),
        y[t] ~ N(B x[t], inv(w_q)), q(x) q(a) q(w_p) q(w_q).  ``a_prior = (ma0, Va0)`` and ``a_init = (E[a], cov(a))`` of
        the initial q(a) (required: an uninformed q(a) makes the first sweep meaningless), in the ABI's row-major order
        a[i * d + j] = A[i, j]: means [d, d] (or [d * d]), covariances [d * d, d * d].  Each noise as for
        :meth:`lgssm_vmp_noise`; both may be known.  d <= 4.  Returns the dict of :meth:`lgssm_vmp_noise` plus
        a_mean[iterations, d, d, batch] and a_cov[iterations, d * d, d * d, batch] after every iteration."""
        self._vmp_dims(y)
        d = np.asarray(S0).shape[-1]
        n = d * d
        if not (isinstance(a_prior, (tuple, list)) and len(a_prior) == 2):
            raise ValueError("a_prior: expected (mean [d, d], covariance [d * d, d * d])")
        if not (isinstance(a_init, (tuple, list)) and len(a_init) == 2):
            raise ValueError("a_init: expected (E[a] [d, d], cov(a) [d * d, d * d]) of the initial q(a)")
        mats = dict(a_mean0=np.asarray(a_prior[0]).reshape(-1), a_cov0=a_prior[1],
                    a_init_mean=np.asarray(a_init[0]).reshape(-1), a_init_cov=a_init[1])
        shapes = dict(a_mean0=(n,), a_cov0=(n, n), a_init_mean=(n,), a_init_cov=(n, n))
        c = self._vmp_setup("lgssm_vmp_transition", y, d, mats, shapes, B, m0, S0, P, p_prior, p_init, Q, q_prior,
                            q_init, u, iterations, mask, transition_first, asynchronous, want_free_energy)
        a_mean, a_cov = self.empty(c.iterations, d, d, c.batch), self.empty(c.iterations, n, n, c.batch)
        self._check(self.lib.rxg_lgssm_vmp_transition_f32(
            *c.head, c.hp("a_mean0"), c.hp("a_cov0"), c.hp("a_init_mean"), c.hp("a_init_cov"), c.hp("B"), c.hp("m0"),
            c.hp("S0"), c.hp("u"), *c.p, *c.q, *c.io, _fp(a_mean), _fp(a_cov), *c.w_out, *c.tail))
        return dict(mean=c.mean, cov=c.cov, a_mean=a_mean, a_cov=a_cov, **c.out, free_energy=c.fe, status=c.st)

    # ------------------------------------------------------------------ per-rule kernels
    def _mat(self, M, name, rows, cols, n):
        """PointMass matrix operand [rows, cols] (None: taken from M): a host array or a CUDA tensor [rows, cols] is one
        matrix shared by every message (shared = 1; a host array is copied to the device), a CUDA tensor [rows, cols, n]
        one matrix per message (shared = 0).  Returns (kept tensor, pointer, shared, (rows, cols))."""
        if isinstance(M, torch.Tensor) and M.is_cuda:
            self._io(M, name)
            shared = M.dim() == 2
            r, c = M.shape[:2] if M.dim() in (2, 3) else (None, None)
            want = (rows or r, cols or c) + (() if shared else (n,))
            if tuple(M.shape) != want:
                raise ValueError(f"{name}: expected a shared CUDA matrix {want[:2]} or one per message {want[:2] + (n,)}, "
                                 f"got {tuple(M.shape)}")
            return M, _fp(M), int(shared), want[:2]
        a = np.ascontiguousarray(np.asarray(M.cpu() if isinstance(M, torch.Tensor) else M, dtype=np.float32))
        if a.ndim != 2 or (rows is not None and a.shape[0] != rows) or (cols is not None and a.shape[1] != cols):
            raise ValueError(f"{name}: expected a host matrix {(rows, cols)} shared by every message, got {a.shape} "
                             f"(a matrix per message is a CUDA tensor [rows, cols, n])")
        t = torch.as_tensor(a, device=f"cuda:{self.device}")
        return t, _fp(t), 1, a.shape

    def _msgs(self, v, name, *mats):
        """A batch of messages: ``v`` [d, n] and the [d, d, n] matrices ``mats`` (name, tensor); returns (d, n)."""
        self._io(v, name, ndim=2)
        d, n = v.shape
        for nm, M in mats:
            self._io(M, nm, shape=(d, d, n))
        return d, n

    def rule_add_cov(self, mu, S, Sigma, which="out"):
        d, n = self._msgs(mu, "mu", ("S", S))
        keep, Sp, shared, _ = self._mat(Sigma, "Sigma", d, d, n)
        mo, So = torch.empty_like(mu), self.empty(d, d, n)
        fn = self.lib.rxg_rule_mvnormal_meancov_out_f32 if which == "out" else self.lib.rxg_rule_mvnormal_meancov_mean_f32
        self._check(fn(self.h, n, d, _fp(mu), _fp(S), Sp, shared, _fp(mo), _fp(So), L.PTR_DEVICE))
        return mo, So

    def rule_mean_from_data(self, y, Sigma):
        d, n = self._msgs(y, "y")
        keep, Sp, shared, _ = self._mat(Sigma, "Sigma", d, d, n)
        mo, So = torch.empty_like(y), self.empty(d, d, n)
        self._check(self.lib.rxg_rule_mvnormal_meancov_mean_data_f32(self.h, n, d, _fp(y), Sp, shared, _fp(mo), _fp(So), L.PTR_DEVICE))
        return mo, So

    def rule_mul_out(self, A, mu, S):
        di, n = self._msgs(mu, "mu", ("S", S))
        keep, Ap, shared, (do, _) = self._mat(A, "A", None, di, n)
        mo, So = self.empty(do, n), self.empty(do, do, n)
        self._check(self.lib.rxg_rule_mul_out_f32(self.h, n, do, di, Ap, shared, _fp(mu), _fp(S), _fp(mo), _fp(So), L.PTR_DEVICE))
        return mo, So

    def rule_mul_in(self, A, mu_out, S_out):
        do, n = self._msgs(mu_out, "mu_out", ("S_out", S_out))
        keep, Ap, shared, (_, di) = self._mat(A, "A", do, None, n)
        xi, W = self.empty(di, n), self.empty(di, di, n)
        st = self.empty(n, dtype=torch.int32)
        self._check(self.lib.rxg_rule_mul_in_f32(self.h, n, do, di, Ap, shared, _fp(mu_out), _fp(S_out), _fp(xi), _fp(W),
                                                 _i32(st), L.PTR_DEVICE))
        return xi, W, st

    def _pair(self, fn, a, Sa, b, Sb):
        d, n = self._msgs(a, "first vector", ("first matrix", Sa), ("second matrix", Sb))
        self._io(b, "second vector", shape=(d, n))
        o, So = torch.empty_like(a), self.empty(d, d, n)
        self._check(fn(self.h, n, d, _fp(a), _fp(Sa), _fp(b), _fp(Sb), _fp(o), _fp(So), L.PTR_DEVICE))
        return o, So

    def rule_add_out(self, mu1, S1, mu2, S2):
        return self._pair(self.lib.rxg_rule_add_out_f32, mu1, S1, mu2, S2)

    def rule_add_in(self, mu_out, S_out, mu_other, S_other):
        return self._pair(self.lib.rxg_rule_add_in_f32, mu_out, S_out, mu_other, S_other)

    def prod_gaussian(self, xi1, W1, xi2, W2):
        return self._pair(self.lib.rxg_prod_gaussian_f32, xi1, W1, xi2, W2)

    def _conv(self, fn, v, M):
        d, n = self._msgs(v, "vector", ("matrix", M))
        vo, Mo = torch.empty_like(v), self.empty(d, d, n)
        st = self.empty(n, dtype=torch.int32)
        self._check(fn(self.h, n, d, _fp(v), _fp(M), _fp(vo), _fp(Mo), _i32(st), L.PTR_DEVICE))
        return vo, Mo, st

    def meancov_to_wmp(self, mu, S):
        return self._conv(self.lib.rxg_meancov_to_wmp_f32, mu, S)

    def wmp_to_meancov(self, xi, W):
        return self._conv(self.lib.rxg_wmp_to_meancov_f32, xi, W)

    def marginal_gaussian(self, msgs):
        """Product of the k (xi [d, n], W [d, d, n]) messages ``msgs``, as (mean, covariance, status)."""
        msgs = list(msgs)
        if not msgs:
            raise ValueError("marginal_gaussian: needs at least one (xi, W) message")
        k = len(msgs)
        d, n = self._msgs(msgs[0][0], "xi[0]", ("W[0]", msgs[0][1]))
        for q, (xi, W) in enumerate(msgs):
            self._io(xi, f"xi[{q}]", shape=(d, n))
            self._io(W, f"W[{q}]", shape=(d, d, n))
        xs = (L.fp * k)(*[_fp(x) for x, _ in msgs])
        ws = (L.fp * k)(*[_fp(w) for _, w in msgs])
        mu, S = self.empty(d, n), self.empty(d, d, n)
        st = self.empty(n, dtype=torch.int32)
        self._check(self.lib.rxg_marginal_gaussian_f32(self.h, n, d, k, xs, ws, _fp(mu), _fp(S),
                                                       _i32(st), L.PTR_DEVICE))
        return mu, S, st

    def _six(self, fn, a, b, c, d_):
        self._dev(a, b, c, d_)
        n = a.numel()
        o1, o2 = torch.empty_like(a), torch.empty_like(a)
        self._check(fn(self.h, n, _fp(a), _fp(b), _fp(c), _fp(d_), _fp(o1), _fp(o2), L.PTR_DEVICE))
        return o1, o2

    def rule_normal_precision_tau(self, m_out, v_out, m_mu, v_mu):
        return self._six(self.lib.rxg_rule_normal_precision_tau_f32, m_out, v_out, m_mu, v_mu)

    def rule_normal_precision_out(self, m_mu, v_mu, shape, rate):
        return self._six(self.lib.rxg_rule_normal_precision_out_f32, m_mu, v_mu, shape, rate)

    def rule_normal_precision_tau_joint(self, m_joint, V_joint):
        """Structured tau rule: q(out, mu) jointly Gaussian, m_joint[2, n], V_joint[2, 2, n]."""
        self._io(m_joint, "m_joint", ndim=2)
        n = m_joint.shape[-1]
        self._io(m_joint, "m_joint", shape=(2, n))
        self._io(V_joint, "V_joint", shape=(2, 2, n))
        sh, rt = self.empty(n), self.empty(n)
        self._check(self.lib.rxg_rule_normal_precision_tau_joint_f32(self.h, n, _fp(m_joint), _fp(V_joint), _fp(sh), _fp(rt), L.PTR_DEVICE))
        return sh, rt

    def rule_mvnormal_precision_lambda(self, m_out, V_out, m_mu, V_mu):
        d, n = self._msgs(m_out, "m_out", ("V_out", V_out), ("V_mu", V_mu))
        self._io(m_mu, "m_mu", shape=(d, n))
        df, iS = self.empty(n), self.empty(d, d, n)
        self._check(self.lib.rxg_rule_mvnormal_precision_lambda_f32(self.h, n, d, _fp(m_out), _fp(V_out), _fp(m_mu), _fp(V_mu),
                                                                    _fp(df), _fp(iS), L.PTR_DEVICE))
        return df, iS

    def _wishart(self, pairs):
        """Wishart messages (df [n], inverse scale [d, d, n]) in ``pairs`` (name, df, iS); returns (d, n)."""
        iS0 = pairs[0][2]
        self._io(iS0, f"{pairs[0][0]}: inverse scale", ndim=3)
        d, n = iS0.shape[0], iS0.shape[-1]
        for name, df, iS in pairs:
            self._io(df, f"{name}: df", shape=(n,))
            self._io(iS, f"{name}: inverse scale", shape=(d, d, n))
        return d, n

    def prod_wishart(self, df1, iS1, df2, iS2):
        d, n = self._wishart([("first", df1, iS1), ("second", df2, iS2)])
        df, iS = self.empty(n), self.empty(d, d, n)
        self._check(self.lib.rxg_prod_wishart_f32(self.h, n, d, _fp(df1), _fp(iS1), _fp(df2), _fp(iS2), _fp(df), _fp(iS), L.PTR_DEVICE))
        return df, iS

    def wishart_mean(self, df, iS):
        d, n = self._wishart([("wishart", df, iS)])
        out = self.empty(d, d, n)
        st = self.empty(n, dtype=torch.int32)
        self._check(self.lib.rxg_wishart_mean_f32(self.h, n, d, _fp(df), _fp(iS), _fp(out),
                                                  _i32(st), L.PTR_DEVICE))
        return out, st

    def mv_iid_wishart_vmp(self, y, iterations=10, mu0=None, Lambda0=None, nu0=None, inv_scale0=None, init_E_P=None):
        """Fused mean-field VMP of the multivariate IID model with Wishart precision (``rxg_mv_iid_wishart_vmp_f32``);
        y[N, d, batch]; defaults = the reference test's priors (mv_iid_precision_tests.jl:10-30)."""
        self._dev(y)
        N, d, batch = y.shape
        mu0 = np.zeros(d) if mu0 is None else mu0
        Lambda0 = 100.0 * np.eye(d) if Lambda0 is None else Lambda0
        nu0 = d + 1.0 if nu0 is None else nu0
        inv_scale0 = np.eye(d) if inv_scale0 is None else inv_scale0
        init_E_P = d * 1e12 * np.eye(d) if init_E_P is None else init_E_P       # mean of vague(Wishart, d)
        keep = [_model32(x) for x in (mu0, Lambda0, inv_scale0, init_E_P)]
        mm, mc = self.empty(d, batch), self.empty(d, d, batch)
        df, iS = self.empty(batch), self.empty(d, d, batch)
        st = self.empty(batch, dtype=torch.int32)
        self._check(self.lib.rxg_mv_iid_wishart_vmp_f32(self.h, d, N, batch, iterations, keep[0][1], keep[1][1], float(nu0),
                                                        keep[2][1], keep[3][1], _fp(y), _fp(mm), _fp(mc), _fp(df), _fp(iS),
                                                        _i32(st), L.PTR_DEVICE))
        return dict(m_mean=mm, m_cov=mc, df=df, inv_scale=iS, status=st)

    def ar_vmp(self, series, order, iterations=15, gamma_prior=(1.0, 1.0), theta_prior_precision=1.0, init_gamma=(1.0, 1.0),
               want_free_energy=True):
        """Fused VMP of the reference's autoregressive regression model (``rxg_ar_vmp_f32``); series[N, batch]."""
        self._dev(series)
        N, batch = series.shape
        tm, tc = self.empty(order, batch), self.empty(order, order, batch)
        gs, gr = self.empty(batch), self.empty(batch)
        fe = self.empty(iterations, batch, dtype=torch.float64) if want_free_energy else None      # fp64 output (see the header)
        self._check(self.lib.rxg_ar_vmp_f32(self.h, order, N, batch, iterations, gamma_prior[0], gamma_prior[1], theta_prior_precision,
                                            init_gamma[0], init_gamma[1], _fp(series), _fp(tm), _fp(tc), _fp(gs),
                                            _fp(gr), _f64(fe), L.PTR_DEVICE))
        return dict(theta_mean=tm, theta_cov=tc, gamma_shape=gs, gamma_rate=gr, free_energy=fe)

    def lar_vmp(self, y, order, tau, iterations=15, gamma_prior=(1.0, 1.0), theta_prior_precision=1.0, x0_prior_precision=1.0,
                init_gamma=(1.0, 1.0), init_theta_precision=1.0, want_states=True, want_free_energy=True):
        """Fused structured VMP of the reference's latent autoregressive model (``rxg_lar_vmp_f32``,
        /root/reference/test/models/autoregressive/lar_tests.jl); y[T, batch] on the device.  Returns the KeepLast
        state posteriors and the KeepEach parameter posteriors / free energy, as the reference's ``returnvars``."""
        self._dev(y)
        if y.dim() != 2:
            raise ValueError("lar_vmp: y must be [T, batch]")
        T, batch = y.shape
        iters = int(iterations)
        prm = (ctypes.c_float * 8)(float(tau), float(gamma_prior[0]), float(gamma_prior[1]), float(theta_prior_precision),
                                   float(x0_prior_precision), float(init_gamma[0]), float(init_gamma[1]), float(init_theta_precision))
        xm = self.empty(T, order, batch) if want_states else None
        xc = self.empty(T, order, order, batch) if want_states else None
        tm, tc = self.empty(iters, order, batch), self.empty(iters, order, order, batch)
        gs, gr = self.empty(iters, batch), self.empty(iters, batch)
        fe = self.empty(iters, batch, dtype=torch.float64) if want_free_energy else None
        st = self.empty(batch, dtype=torch.int32)
        self._check(self.lib.rxg_lar_vmp_f32(self.h, int(order), T, batch, iters, ctypes.cast(prm, L.fp), _fp(y), _fp(xm), _fp(xc),
                                             _fp(tm), _fp(tc), _fp(gs), _fp(gr), _f64(fe),
                                             _i32(st), L.PTR_DEVICE))
        return dict(x_mean=xm, x_cov=xc, theta_mean=tm, theta_cov=tc, gamma_shape=gs, gamma_rate=gr, free_energy=fe, status=st)

    def gmm_vmp(self, y, alpha0, mu0, V0, nu0, S0, alpha_init, m_init, Vm_init, nu_init, S_init, iterations=10,
                want_free_energy=True, want_z=False, keep_each=False):
        """Fused mean-field VMP of the Gaussian mixture model (``rxg_gmm_vmp_f32``); y[N, d, batch] on the device.
        Priors and initial marginals are host arrays shared by every chain: alpha0[K], mu0[K, d], V0[K, d, d] (covariance),
        nu0[K], S0[K, d, d] (Wishart scale); the same for the initial q(s), q(m), q(W).  Returns the last iteration's
        ``alpha[K, batch]``, ``m_mean[K, d, batch]``, ``m_cov[K, d, d, batch]``, ``w_df[K, batch]``,
        ``w_inv_scale[K, d, d, batch]``, ``free_energy[iterations, batch]`` (fp64), ``z_prob[N, K, batch]`` (with
        ``want_z``), ``status[batch]`` and, with ``keep_each``, ``hist_*`` with a leading iteration axis."""
        self._dev(y)
        if y.dim() != 3:
            raise ValueError("gmm_vmp: y must be [N, d, batch]")
        N, d, batch = y.shape
        K = int(np.asarray(alpha0).shape[0])
        keep = _host_arrays("gmm_vmp", dict(alpha0=(alpha0, (K,)), mu0=(mu0, (K, d)), V0=(V0, (K, d, d)),
                                            nu0=(nu0, (K,)), S0=(S0, (K, d, d)), alpha_init=(alpha_init, (K,)),
                                            m_init=(m_init, (K, d)), Vm_init=(Vm_init, (K, d, d)),
                                            nu_init=(nu_init, (K,)), S_init=(S_init, (K, d, d))), f"K = {K}, d = {d}")
        its = int(iterations)
        al, mm, mc = self.empty(K, batch), self.empty(K, d, batch), self.empty(K, d, d, batch)
        df, iS = self.empty(K, batch), self.empty(K, d, d, batch)
        fe = self.empty(its, batch, dtype=torch.float64) if want_free_energy else None
        z = self.empty(N, K, batch) if want_z else None
        h = dict(hist_alpha=self.empty(its, K, batch), hist_m_mean=self.empty(its, K, d, batch),
                 hist_m_cov=self.empty(its, K, d, d, batch), hist_w_df=self.empty(its, K, batch),
                 hist_w_inv_scale=self.empty(its, K, d, d, batch)) if keep_each else {}
        st = self.empty(batch, dtype=torch.int32)
        self._check(self.lib.rxg_gmm_vmp_f32(self.h, d, K, N, batch, its, *(p for _, p in keep.values()), _fp(y),
                                             _fp(al), _fp(mm), _fp(mc), _fp(df), _fp(iS), _f64(fe), _fp(z),
                                             *(_fp(h.get(k)) for k in ("hist_alpha", "hist_m_mean", "hist_m_cov",
                                                                         "hist_w_df", "hist_w_inv_scale")),
                                             _i32(st), L.PTR_DEVICE))
        out = dict(alpha=al, m_mean=mm, m_cov=mc, w_df=df, w_inv_scale=iS, free_energy=fe, z_prob=z, status=st)
        out.update(h)
        return out

    def hmm_vmp(self, x, p0, A_prior=None, A_init=None, A_known=None, B_prior=None, B_init=None, B_known=None,
                iterations=1, want_free_energy=True, keep_each=False):
        """Fused structured VMP of the hidden Markov model (``rxg_hmm_vmp_f32``); x[T, batch] uint8 symbols on the device
        (255 = missing).  p0[K] and each matrix are host arrays shared by every chain, columns = conditionals: A learned
        (``A_prior`` and ``A_init``, Dirichlet parameters [K, K]) or known (``A_known``, a probability matrix); B likewise
        with shape [M, K].  Returns ``s_prob[T, K, batch]``, ``s0_prob[K, batch]``, ``A_alpha[K, K, batch]`` /
        ``B_alpha[M, K, batch]`` (None when known), ``free_energy[iterations, batch]`` (fp64), ``status[batch]`` and, with
        ``keep_each``, ``hist_s`` / ``hist_A`` / ``hist_B`` with a leading iteration axis."""
        self._io(x, "hmm_vmp: x [T, batch]", dtype=torch.uint8, ndim=2)
        T, batch = x.shape
        K = int(np.asarray(p0).reshape(-1).shape[0])
        B_any = B_known if B_known is not None else B_prior
        if B_any is None:
            raise ValueError("hmm_vmp: pass either B_prior and B_init (B learned) or B_known")
        M = int(np.asarray(B_any).shape[0])
        keep = _host_arrays("hmm_vmp", dict(p0=(p0, (K,)), A_prior=(A_prior, (K, K)), A_init=(A_init, (K, K)),
                                            A_known=(A_known, (K, K)), B_prior=(B_prior, (M, K)),
                                            B_init=(B_init, (M, K)), B_known=(B_known, (M, K))),
                            f"K = {K}, M = {M}", nulls=True)
        learn_A, learn_B = A_known is None, B_known is None
        its = int(iterations)
        sp, s0 = self.empty(T, K, batch), self.empty(K, batch)
        Aa = self.empty(K, K, batch) if learn_A else None
        Ba = self.empty(M, K, batch) if learn_B else None
        fe = self.empty(its, batch, dtype=torch.float64) if want_free_energy else None
        h = {}
        if keep_each:
            h["hist_s"] = self.empty(its, T, K, batch)
            h["hist_A"] = self.empty(its, K, K, batch) if learn_A else None
            h["hist_B"] = self.empty(its, M, K, batch) if learn_B else None
        st = self.empty(batch, dtype=torch.int32)
        self._check(self.lib.rxg_hmm_vmp_f32(self.h, K, M, T, batch, its, *(p for _, p in keep.values()), _u8(x),
                                             _fp(sp), _fp(s0), _fp(Aa), _fp(Ba), _f64(fe), _fp(h.get("hist_s")),
                                             _fp(h.get("hist_A")), _fp(h.get("hist_B")), _i32(st), L.PTR_DEVICE))
        out = dict(s_prob=sp, s0_prob=s0, A_alpha=Aa, B_alpha=Ba, free_energy=fe, status=st)
        out.update(h)
        return out

    def hmm_gauss_vmp(self, y, p0, mu0, V0, nu0, S0, m_init, Vm_init, nu_init, S_init, A_prior=None, A_init=None,
                      A_known=None, iterations=1, want_free_energy=True, keep_each=False):
        """Fused structured VMP of the hidden Markov model with Gaussian emissions (``rxg_hmm_gauss_vmp_f32``); y[T, d, batch]
        on the device (an all-NaN step is missing).  p0[K], A (learned: ``A_prior`` and ``A_init``, Dirichlet parameters
        [K, K]; known: ``A_known``, a probability matrix; columns = conditionals) and the emission priors and initial
        marginals (mu0[K, d], V0[K, d, d] covariance, nu0[K], S0[K, d, d] Wishart scale; likewise m_init, Vm_init, nu_init,
        S_init) are host arrays shared by every chain.  Returns ``s_prob[T, K, batch]``, ``s0_prob[K, batch]``,
        ``A_alpha[K, K, batch]`` (None when known), ``m_mean[K, d, batch]``, ``m_cov[K, d, d, batch]``, ``w_df[K, batch]``,
        ``w_inv_scale[K, d, d, batch]``, ``free_energy[iterations, batch]`` (fp64), ``status[batch]`` and, with
        ``keep_each``, ``hist_*`` with a leading iteration axis."""
        self._dev(y)
        if y.dim() != 3:
            raise ValueError("hmm_gauss_vmp: y must be [T, d, batch]")
        T, d, batch = y.shape
        K = int(np.asarray(p0).reshape(-1).shape[0])
        vals = dict(p0=(p0, (K,)), A_prior=(A_prior, (K, K)), A_init=(A_init, (K, K)), A_known=(A_known, (K, K)),
                    mu0=(mu0, (K, d)), V0=(V0, (K, d, d)), nu0=(nu0, (K,)), S0=(S0, (K, d, d)), m_init=(m_init, (K, d)),
                    Vm_init=(Vm_init, (K, d, d)), nu_init=(nu_init, (K,)), S_init=(S_init, (K, d, d)))
        keep = _host_arrays("hmm_gauss_vmp", vals, f"K = {K}, d = {d}", nulls=True)
        learn_A = A_known is None
        its = int(iterations)
        sp, s0 = self.empty(T, K, batch), self.empty(K, batch)
        Aa = self.empty(K, K, batch) if learn_A else None
        mm, mc, df, iS = self.empty(K, d, batch), self.empty(K, d, d, batch), self.empty(K, batch), self.empty(K, d, d, batch)
        fe = self.empty(its, batch, dtype=torch.float64) if want_free_energy else None
        h = dict(hist_s=self.empty(its, T, K, batch), hist_A=self.empty(its, K, K, batch) if learn_A else None,
                 hist_m_mean=self.empty(its, K, d, batch), hist_m_cov=self.empty(its, K, d, d, batch),
                 hist_w_df=self.empty(its, K, batch), hist_w_inv_scale=self.empty(its, K, d, d, batch)) if keep_each else {}
        st = self.empty(batch, dtype=torch.int32)
        self._check(self.lib.rxg_hmm_gauss_vmp_f32(self.h, d, K, T, batch, its, *(p for _, p in keep.values()), _fp(y),
                                                   _fp(sp), _fp(s0), _fp(Aa), _fp(mm), _fp(mc), _fp(df), _fp(iS),
                                                   _f64(fe),
                                                   *(_fp(h.get(k)) for k in ("hist_s", "hist_A", "hist_m_mean", "hist_m_cov",
                                                                               "hist_w_df", "hist_w_inv_scale")),
                                                   _i32(st), L.PTR_DEVICE))
        out = dict(s_prob=sp, s0_prob=s0, A_alpha=Aa, m_mean=mm, m_cov=mc, w_df=df, w_inv_scale=iS, free_energy=fe, status=st)
        out.update(h)
        return out

    def binomial_polya_vmp(self, X, y, xi0, W0, ntrials=None, iterations=1, want_free_energy=True, keep_each=False):
        """Bayesian binomial / logistic regression by mean-field Polya-Gamma VMP (``rxg_binomial_polya_vmp_f32``), one chain
        per batch column: X[N, p, batch] float32, y[N, batch] and ntrials[N, batch] (None: every n = 1) int32 on the
        device; xi0[p] and W0[p, p] (the prior's weighted mean and precision) are host arrays shared by every chain.  A
        sample with n = 0 contributes nothing.  Returns ``beta_mean[p, batch]``, ``beta_cov[p, p, batch]``,
        ``free_energy[iterations, batch]`` (fp64), ``status[batch]`` and, with ``keep_each``, ``hist_mean`` / ``hist_cov``
        with a leading iteration axis."""
        self._dev(X)
        if X.dim() != 3:
            raise ValueError("binomial_polya_vmp: X must be [N, p, batch]")
        N, p, batch = X.shape
        if y is None:
            raise ValueError("binomial_polya_vmp: y is required")
        self._io(y, "binomial_polya_vmp: y [N, batch]", dtype=torch.int32, shape=(N, batch))
        self._io(ntrials, "binomial_polya_vmp: ntrials [N, batch]", dtype=torch.int32, shape=(N, batch))
        keep = _host_arrays("binomial_polya_vmp", dict(xi0=(xi0, (p,)), W0=(W0, (p, p))), f"p = {p}")
        its = int(iterations)
        mean, cov = self.empty(p, batch), self.empty(p, p, batch)
        fe = self.empty(its, batch, dtype=torch.float64) if want_free_energy else None
        h = dict(hist_mean=self.empty(its, p, batch), hist_cov=self.empty(its, p, p, batch)) if keep_each else {}
        st = self.empty(batch, dtype=torch.int32)
        self._check(self.lib.rxg_binomial_polya_vmp_f32(self.h, p, N, batch, its, keep["xi0"][1], keep["W0"][1], _fp(X),
                                                        _i32(y), _i32(ntrials), _fp(mean), _fp(cov), _f64(fe),
                                                        _fp(h.get("hist_mean")), _fp(h.get("hist_cov")), _i32(st),
                                                        L.PTR_DEVICE))
        out = dict(beta_mean=mean, beta_cov=cov, free_energy=fe, status=st)
        out.update(h)
        return out

    def _multinomial_args(self, who, y, xi0, W0):
        """y: a contiguous int32 CUDA tensor [n, K, batch] on this context's device; the prior (xi0 [D], W0 [D, D], D = K - 1)
        as the fp32 host arrays the C entries take."""
        self._io(y, f"{who}: y [n, K, batch]", dtype=torch.int32, ndim=3)
        D = y.shape[1] - 1
        return D, _host_arrays(who, dict(xi0=(xi0, (D,)), W0=(W0, (D, D))), f"K = {D + 1}")

    def multinomial_polya_vmp(self, y, xi0, W0, iterations=1, want_free_energy=True, keep_each=False):
        """Bayesian multinomial regression by mean-field Polya-Gamma VMP over whole data sets
        (``rxg_multinomial_polya_vmp_f32``), one chain per batch column: counts y[n, K, batch] int32 on the device (an
        all-zero sample contributes nothing); xi0[D] and W0[D, D] (the prior's weighted mean and precision, D = K - 1) are
        host arrays shared by every chain.  Returns ``psi_mean[D, batch]``, ``psi_cov[D, D, batch]``,
        ``free_energy[iterations, batch]`` (fp64), ``status[batch]`` and, with ``keep_each``, ``hist_mean`` / ``hist_cov``
        with a leading iteration axis."""
        D, keep = self._multinomial_args("multinomial_polya_vmp", y, xi0, W0)
        n, K, batch = y.shape
        its = int(iterations)
        mean, cov = self.empty(D, batch), self.empty(D, D, batch)
        fe = self.empty(its, batch, dtype=torch.float64) if want_free_energy else None
        h = dict(hist_mean=self.empty(its, D, batch), hist_cov=self.empty(its, D, D, batch)) if keep_each else {}
        st = self.empty(batch, dtype=torch.int32)
        self._check(self.lib.rxg_multinomial_polya_vmp_f32(self.h, K, n, batch, its, keep["xi0"][1], keep["W0"][1],
                                                           _i32(y), _fp(mean), _fp(cov), _f64(fe), _fp(h.get("hist_mean")),
                                                           _fp(h.get("hist_cov")), _i32(st), L.PTR_DEVICE))
        out = dict(psi_mean=mean, psi_cov=cov, free_energy=fe, status=st)
        out.update(h)
        return out

    def multinomial_polya_online(self, y, xi0, W0, m=None, S=None, iterations=1, want_free_energy=True,
                                 keep_mean=True, keep_cov=True, in_place=False):
        """The same model online (``rxg_multinomial_polya_online_f32``): datum t of y[T, K, batch] (int32, device) runs
        ``iterations`` steps from q_{t-1}.  The carry is fp64 on the device, m[D, batch] and S[D, D, batch]; None starts
        every chain at the prior (xi0, W0).  ``in_place`` updates the given carry.  Returns ``m``, ``S`` (the carry after
        the last datum), ``hist_mean[T, D, batch]`` / ``hist_cov[T, D, D, batch]`` (None when not kept),
        ``free_energy[T, batch]`` (fp64, per datum) and ``status[batch]``."""
        D, keep = self._multinomial_args("multinomial_polya_online", y, xi0, W0)
        T, K, batch = y.shape
        if (m is None) != (S is None):
            raise ValueError("multinomial_polya_online: pass the carry m and S together, or neither")
        self._io(m, "multinomial_polya_online: m [D, batch]", dtype=torch.float64, shape=(D, batch))
        self._io(S, "multinomial_polya_online: S [D, D, batch]", dtype=torch.float64, shape=(D, D, batch))
        if in_place and m is None:
            raise ValueError("multinomial_polya_online: in_place needs a carry")
        m_out = m if in_place else self.empty(D, batch, dtype=torch.float64)
        S_out = S if in_place else self.empty(D, D, batch, dtype=torch.float64)
        hm = self.empty(T, D, batch) if keep_mean else None
        hc = self.empty(T, D, D, batch) if keep_cov else None
        fe = self.empty(T, batch, dtype=torch.float64) if want_free_energy else None
        st = self.empty(batch, dtype=torch.int32)
        self._check(self.lib.rxg_multinomial_polya_online_f32(self.h, K, T, batch, int(iterations), keep["xi0"][1],
                                                              keep["W0"][1], _f64(m), _f64(S), _i32(y), _f64(m_out),
                                                              _f64(S_out), _fp(hm), _fp(hc), _f64(fe), _i32(st),
                                                              L.PTR_DEVICE))
        return dict(m=m_out, S=S_out, hist_mean=hm, hist_cov=hc, free_energy=fe, status=st)

    def prod_gamma(self, a1, b1, a2, b2):
        return self._six(self.lib.rxg_prod_gamma_f32, a1, b1, a2, b2)

    def prod_normal(self, m1, v1, m2, v2):
        return self._six(self.lib.rxg_prod_normal_f32, m1, v1, m2, v2)

    def rule_gcv_out(self, m_x, v_x, m_z, v_z, kappa, omega):
        self._dev(m_x, v_x, m_z, v_z)
        n = m_x.numel()
        mo, vo = torch.empty_like(m_x), torch.empty_like(m_x)
        self._check(self.lib.rxg_rule_gcv_out_f32(self.h, n, _fp(m_x), _fp(v_x), _fp(m_z), _fp(v_z), kappa, omega, _fp(mo), _fp(vo), L.PTR_DEVICE))
        return mo, vo

    def marginalrule_gcv_yx(self, m_y, v_y, m_x, v_x, m_z, v_z, kappa, omega):
        self._dev(m_y, v_y, m_x, v_x, m_z, v_z)
        n = m_y.numel()
        m, V = self.empty(2, n), self.empty(2, 2, n)
        self._check(self.lib.rxg_marginalrule_gcv_yx_f32(self.h, n, _fp(m_y), _fp(v_y), _fp(m_x), _fp(v_x), _fp(m_z), _fp(v_z),
                                                         kappa, omega, _fp(m), _fp(V), L.PTR_DEVICE))
        return m, V

    def rule_gcv_z_prod(self, m_yx, V_yx, m_zp, v_zp, kappa, omega):
        self._dev(m_yx, V_yx, m_zp, v_zp)
        n = m_zp.numel()
        mz, vz = torch.empty_like(m_zp), torch.empty_like(m_zp)
        self._check(self.lib.rxg_rule_gcv_z_prod_f32(self.h, n, _fp(m_yx), _fp(V_yx), _fp(m_zp), _fp(v_zp), kappa, omega,
                                                     _fp(mz), _fp(vz), L.PTR_DEVICE))
        return mz, vz

    def selftest_umma(self, A, B):
        """D[128, n] = A[128, k] @ B[n, k].T on the tensor cores (wgmma, 3xTF32), for the sweeps' operand shapes."""
        self._dev(A, B)
        n, k = B.shape
        D = self.empty(128, n)
        self._check(self.lib.rxg_selftest_umma_shape_f32(self.h, n, k, _fp(A), _fp(B), _fp(D), L.PTR_DEVICE))
        return D

    def selftest_stream(self, src, dst, asynchronous=True):
        """dst[w, :] = sum_r src[r, :] -- streaming kernel with a (n_read : n_write) HBM traffic mix."""
        nr, n = src.shape
        nw = dst.shape[0]
        self._dev(src if nr else None, dst if nw else None)
        self._check(self.lib.rxg_selftest_stream_f32(self.h, n, nr, nw, _fp(src), _fp(dst),
                                                     L.PTR_DEVICE | (L.ASYNC if asynchronous else 0)))
        return dst

    # ------------------------------------------------------------------ multi-GPU
    def comm_init(self, nranks, rank, uid: bytes):
        buf = ctypes.create_string_buffer(uid, 128)
        self._check(self.lib.rxg_comm_init(self.h, nranks, rank, ctypes.cast(buf, c_void_p)))
        self.comm_nranks, self.comm_rank = int(nranks), int(rank)

    # ---- peer-mapped gather (NVLink P2P stores from the sweep itself; rxg_peer.cu)
    def peer_open(self, handle: bytes) -> int:
        buf = ctypes.create_string_buffer(handle, 64)
        p = c_void_p()
        self._check(self.lib.rxg_peer_open(self.h, ctypes.cast(buf, c_void_p), ctypes.byref(p)))
        return int(p.value)

    def peer_close(self, ptr: int):
        self._check(self.lib.rxg_peer_close(self.h, c_void_p(ptr)))

    def peer_group(self, nranks: int, rank: int, flag_ptrs):
        arr = (c_void_p * max(nranks, 1))(*[c_void_p(int(p)) for p in flag_ptrs]) if nranks > 1 else None
        self._check(self.lib.rxg_peer_group(self.h, nranks, rank, arr))
        self.peer_nranks, self.peer_rank = int(nranks), int(rank)

    def peer_barrier(self, asynchronous=False):
        self._check(self.lib.rxg_peer_barrier(self.h, L.ASYNC if asynchronous else 0))

    def peer_allgather(self, local, gathered_ptrs, asynchronous=False):
        """``local`` (contiguous CUDA fp32) -> slab ``rank`` of every rank's gathered buffer, then the barrier."""
        self._dev(local)
        arr = (L.fp * len(gathered_ptrs))(*[L.as_fp(p) for p in gathered_ptrs])
        self._check(self.lib.rxg_peer_allgather_f32(self.h, local.numel(), _fp(local), arr,
                                                    L.PTR_DEVICE | (L.ASYNC if asynchronous else 0)))

    def lgssm_smooth_gather(self, y, A, B, P, Q, m0, S0, gathered_mean_ptrs, gathered_cov_ptrs=None, *, u=None, mask=None,
                            replicate_cov=False, want_evidence=False, want_status=False, force_per_chain_path=False,
                            transition_first=False, asynchronous=False):
        """Fused smoothing sweep + all-gather (``rxg_lgssm_smooth_gather_f32``).  ``gathered_*_ptrs[g]`` = base address
        of rank g's gathered buffer as mapped in this process (see ``sharding.PeerGroup``)."""
        self._io(y, "y", True)
        T, m, batch = y.shape
        self._io(mask, "mask", True, dtype=torch.uint8, shape=(T, batch))
        d = np.asarray(A).shape[-1]
        keep = [_model32(x) for x in (A, B, P, Q, m0, S0)]
        ptrs = [k[1] for k in keep]
        if u is not None:
            keep.append(_model32(u)); ptrs.append(keep[-1][1])
        else:
            ptrs.append(L.as_fp(0))
        flags = L.PTR_DEVICE
        if replicate_cov:
            flags |= L.COV_REPLICATE
        if force_per_chain_path:
            flags |= L.PATH_PER_CHAIN
        if transition_first:
            flags |= L.TRANSITION_FIRST
        if asynchronous:
            flags |= L.ASYNC
        G = len(gathered_mean_ptrs)
        gm = (L.fp * G)(*[L.as_fp(p) for p in gathered_mean_ptrs])
        gc = (L.fp * G)(*[L.as_fp(p) for p in gathered_cov_ptrs]) if gathered_cov_ptrs is not None else None
        nle = self.empty(batch) if want_evidence else None
        status = self.empty(batch, dtype=torch.int32) if want_status else None
        mask_p = ctypes.cast(c_void_p(mask.data_ptr() if mask is not None else None), L.u8p)
        st_p = ctypes.cast(c_void_p(status.data_ptr() if status is not None else None), L.i32p)
        self._check(self.lib.rxg_lgssm_smooth_gather_f32(self.h, d, m, T, batch, *ptrs, _fp(y), mask_p, gm, gc, _fp(nle), st_p, flags))
        return dict(neg_log_evidence=nle, status=status)

    def allgather_posteriors(self, mean, cov, nranks, out_mean=None, out_cov=None, replicate_cov=False):
        """Rank-major gathered slabs ([G, T, d, b], [G, T, d, d, b]); pass out_* to reuse buffers.
        ``replicate_cov=True`` (shared model on every rank, no missing data: chain-independent
        covariances): only the means cross NVLink, the covariance slabs are filled locally;
        ``cov`` may then also be the de-duplicated [T, d, d] table of ``cov_shared_out=True``."""
        self._dev(mean, cov)
        T, d, bl = mean.shape
        gm = out_mean if out_mean is not None else self.empty(nranks, T, d, bl)
        gc = None
        flags = L.PTR_DEVICE
        if cov is not None:
            gc = out_cov if out_cov is not None else self.empty(nranks, T, d, d, bl)
            if replicate_cov:
                flags |= L.COV_REPLICATE
                if cov.dim() == 3:
                    flags |= L.COV_SHARED_OUT
            elif cov.dim() == 3:
                raise ValueError("a [T, d, d] covariance table can only be replicated (replicate_cov=True)")
        self._check(self.lib.rxg_allgather_posteriors(self.h, d, T, bl, _fp(mean), _fp(cov), _fp(gm), _fp(gc), flags))
        return gm, gc


def host_empty(*shape, dtype=torch.float32):
    """Pinned host tensor from ``rxg_host_alloc`` -- what a C / Julia host of the ABI would use: page-locked and, on a
    multi-socket machine, interleaved over the NUMA nodes (see rxg_api.cu).  Freed when the tensor is collected."""
    lib = L.load()
    n = int(np.prod(shape))
    item = torch.empty((), dtype=dtype).element_size()
    p = c_void_p()
    rc = lib.rxg_host_alloc(ctypes.byref(p), max(n * item, 1))
    if rc != 0:
        raise L.RxGaussError(rc, "rxg_host_alloc failed")
    buf = (ctypes.c_char * (n * item)).from_address(p.value)
    t = torch.frombuffer(buf, dtype=dtype, count=n).reshape(*shape)
    import weakref
    weakref.finalize(buf, lib.rxg_host_free, c_void_p(p.value))
    t._rxg_keep = buf
    return t


class DeviceBuffer:
    """Device memory from ``rxg_device_alloc`` (plain cudaMalloc: exportable as a CUDA IPC handle at offset 0),
    viewable as a torch tensor through ``__cuda_array_interface__``.  Freed with the object."""

    def __init__(self, ctx: "Context", nbytes: int, zero: bool = False):
        self.ctx, self.nbytes = ctx, int(nbytes)
        p = c_void_p()
        ctx._check(ctx.lib.rxg_device_alloc(ctx.h, self.nbytes, ctypes.byref(p)))
        self.ptr = int(p.value)
        if zero:
            ctx._check(ctx.lib.rxg_device_memset(ctx.h, c_void_p(self.ptr), 0, self.nbytes))

    def export(self) -> bytes:
        buf = ctypes.create_string_buffer(64)
        self.ctx._check(self.ctx.lib.rxg_peer_export(self.ctx.h, c_void_p(self.ptr), ctypes.cast(buf, c_void_p)))
        return buf.raw

    def tensor(self, *shape, dtype=torch.float32):
        n = int(np.prod(shape))
        itemsize = torch.empty((), dtype=dtype).element_size()
        assert n * itemsize <= self.nbytes
        typestr = {torch.float32: "<f4", torch.int32: "<i4", torch.uint8: "|u1"}[dtype]
        holder = type("_CAI", (), {})()
        holder.__cuda_array_interface__ = {"shape": tuple(int(x) for x in shape), "typestr": typestr,
                                           "data": (self.ptr, False), "version": 2, "strides": None}
        holder._keep = self
        return torch.as_tensor(holder, device=f"cuda:{self.ctx.device}")

    def free(self):
        if getattr(self, "ptr", None) and getattr(self.ctx, "h", None):
            self.ctx.lib.rxg_device_free(self.ctx.h, c_void_p(self.ptr))
        self.ptr = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


def comm_unique_id() -> bytes:
    lib = L.load()
    buf = ctypes.create_string_buffer(128)
    rc = lib.rxg_comm_unique_id(ctypes.cast(buf, c_void_p))
    if rc != 0:
        raise L.RxGaussError(rc, "rxg_comm_unique_id failed")
    return buf.raw
