"""The large-state LGSSM family (d = m in {8, 16, 32, 64}: csrc/rxg_lgssm_large.cu, csrc/rxg_umma_sweep.cu), chain by
chain, against a plain fp64 Kalman filter + RTS smoother.

The family computes the chain-independent covariances, gains and evidence constants once in fp64 (forward by doubling
and a backward suffix scan, or sequentially with ``large_seq``), then runs the per-chain means through one of two
sweeps: the FP32-pipe block sweep (32 chains per CTA; always at d = 8, ``no_umma`` at d >= 16) or the tensor-core sweep
(64 chains per CTA, wgmma 3xTF32, after a time-sliced ``K_t y_t`` pre-pass).  The evidence is a separate time-sliced
kernel over the filtered means.  Every shape outside the register families (d or m > 6) is embedded into it.

The tests gate EVERY chain (not a norm over the batch) and the covariance table at EVERY step, so that an error confined
to one chain tile, one time slice or one doubling round cannot hide in the healthy rest, and they run the launch
geometries that matter -- the pre-pass and evidence slices are cut from the device's SM count (``launch_geometry``) --
up to BASELINE configs[2] itself (d = 64, T = 1000, 4096 chains).  The reference is the one of
test_shared_sweep_variants.py (textbook, shape agnostic, checked against the oracle below at 1e-10).
"""
import itertools

import numpy as np
import pytest
import torch

from oracle import lgssm
from test_shared_sweep_variants import (WORST, _record, covariance_side, gate_mean, gate_nle, offset, pattern,
                                        random_model, reference_sweep, simulate)
from util import TOL_COV, f32_model

NATIVE_D = [8, 16, 32, 64]
# general shapes and the large-state family they are embedded into (embedding_shape in rxg_lgssm_general.cu)
EMBEDDED = {(7, 7): 8, (9, 4): 16, (2, 9): 16, (12, 7): 16, (24, 24): 32, (33, 20): 64, (64, 32): 64}
CAT = "large-state "        # prefix of this module's categories in the shared per-chain worst-case table


def native_model(d, bkind):
    """``I``: configs[2]'s dense model (A = 0.99 Orth, B = I: the family skips both B products); ``dense``: a
    random model with a dense B (Q >= 1.5 I keeps the per-chain evidence gate meaningful)."""
    if bkind == "I":
        return f32_model(lgssm.dense_model(d, seed=64 + d))
    return random_model(d, d, seed=5000 + d)


def _kw(mod):
    return dict(A=mod["A"], B=mod["B"], P=mod["P"], Q=mod["Q"], m0=mod["m0"], S0=mod["S0"])


# ====================================================================================== launch geometry
SWEEP_ROWS, BLOCK_NB, EV_NB = 64, 32, 32      # chains per CTA: wgmma sweep, block sweep, evidence kernel


def _cdiv(a, b):
    return -(-a // b)


def _slice_steps(T, n):
    """Lengths of the n time slices a kernel cuts [0, T) into (t_lo = T * i / n)."""
    return sorted({T * (i + 1) // n - T * i // n for i in range(n)})


def launch_geometry(sm, T, batch):
    """The grids of the large-state family, restated from an SM count: ``launch_umma_sweep_d`` (wgmma sweep tiles and
    the ``tsplit`` time slices of its K_t y_t pre-pass, about two CTAs per SM) and ``run_large`` (the evidence
    kernel's tiles and ``ev_slices`` time slices, about four CTAs per SM).  ``*_steps`` = the distinct slice lengths."""
    tiles = _cdiv(batch, SWEEP_ROWS)
    tsplit = min(max(_cdiv(2 * sm, tiles), 1), T)
    ev_tiles = _cdiv(batch, EV_NB)
    ev_slices = min(max(_cdiv(4 * sm, ev_tiles), 1), T)
    return dict(tiles=tiles, tsplit=tsplit, ky_steps=_slice_steps(T, tsplit), block_tiles=_cdiv(batch, BLOCK_NB),
                ev_tiles=ev_tiles, ev_slices=ev_slices, ev_steps=_slice_steps(T, ev_slices))


def batch_for(sm, T, pred, lo=1, hi=1 << 16):
    """Smallest batch in [lo, hi) whose geometry satisfies ``pred``."""
    for b in range(lo, hi):
        if pred(launch_geometry(sm, T, b)):
            return b
    raise AssertionError("no batch reaches the requested geometry")


def sm_count():
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


# ====================================================================================== per-step covariance gate
def gate_cov_steps(cat, case, cov, ref_tab, tol=TOL_COV, identical=True):
    """``cov`` per chain [T, d, d, batch] or the table [T, d, d], gated step by step: the largest relative Frobenius
    error over t must meet ``tol``, so an error at one doubling round or suffix-scan boundary cannot hide in a T-long
    norm.  Per chain with ``identical`` (the gain-table path): every chain must hold chain 0's table bit for bit;
    without it (the per-chain kernel) every chain is gated on its own."""
    if cov.dim() == 4 and identical:
        for t0 in range(0, cov.shape[0], 8):
            blk = cov[t0:t0 + 8]
            bad = (~(blk == blk[..., :1]).flatten(0, 2).all(0)).nonzero()
            assert bad.numel() == 0, f"{case}: covariance of chain {int(bad[0])} differs from chain 0 (steps >= {t0})"
    g = (cov[..., :1] if identical else cov) if cov.dim() == 4 else cov[..., None]
    g = g.to("cpu", torch.float64).flatten(1, 2)                                    # [T, d * d, chains]
    r = torch.as_tensor(np.asarray(ref_tab), dtype=torch.float64).flatten(1)[..., None]
    err = torch.nan_to_num((g - r).norm(dim=1) / r.norm(dim=1), nan=float("inf"))  # [T, chains]
    t, b = divmod(int(err.argmax()), err.shape[1]); e = float(err[t, b])
    _record(cat + " cov/step", e, f"{case}, step {t}", b if cov.dim() == 4 and not identical else -1)
    assert e < tol, f"{case}: covariance relative Frobenius at step {t} (chain {b}) = {e:.3e} >= {tol:g}"
    return e


def _eq(a, b, what, case):
    if a is None and b is None:
        return
    assert a is not None and b is not None and torch.equal(a, b), f"{case}: {what} not bit-identical"


@pytest.fixture(scope="module", autouse=True)
def _report_worst():
    yield
    mine = sorted(k for k in WORST if k.startswith(CAT))
    if mine:
        print("\nlarge-state family, per-chain worst cases:")
        for cat in mine:
            e, case, b = WORST.pop(cat)
            print(f"  {cat[len(CAT):]:<28s} {e:.3e}  ({case}, chain {b})")


# ====================================================================================== CPU: the reference itself
CPU_SHAPES = [(8, 8, "I"), (8, 8, "dense"), (16, 16, "I"), (16, 16, "dense"), (12, 7, "dense"), (2, 9, "dense")]


def _cpu_model(d, m, bkind):
    return native_model(d, bkind) if d == m else random_model(d, m, seed=6000 + 16 * d + m)


def _rel(a, b):
    a = np.asarray(a, np.float64); b = np.asarray(b, np.float64)
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-300))


@pytest.mark.parametrize("d,m,bkind", CPU_SHAPES)
@pytest.mark.parametrize("case", ["plain", "offset", "offset_tf", "mask", "mu0"])
def test_reference_matches_oracle(d, m, bkind, case):
    """The fp64 reference at the family's shapes (B = I and dense) and at two embedded originals, against the oracle's
    message schedule and textbook smoother (1e-10): offset, prior one transition earlier, per-chain prior means and a
    shared missing-data pattern."""
    mod = _cpu_model(d, m, bkind)
    T, batch = 30, 5
    y = simulate(mod, T, batch, seed=d + 3 * m)
    u, tf, tm, mu0 = None, False, None, None
    if case in ("offset", "offset_tf"):
        u, tf = offset(d, d + m).astype(np.float64), case == "offset_tf"
    elif case == "mask":
        tm = pattern(T)
    elif case == "mu0":
        mu0 = np.random.default_rng(d * m).standard_normal((d, batch))
    omod = dict(mod) if mu0 is None else dict(mod, m0=mu0.T.copy())
    full = None if tm is None else np.repeat(tm[:, None], batch, axis=1)
    cs = covariance_side(mod, T, tm, tf)
    mu0t = None if mu0 is None else torch.as_tensor(mu0)
    sm = reference_sweep(mod, torch.as_tensor(y), smooth=True, u=u, mu0=mu0t, cs=cs)
    fl = reference_sweep(mod, torch.as_tensor(y), smooth=False, u=u, mu0=mu0t, cs=cs)
    for ref in (lgssm.smooth_reference_schedule(y, **omod, mask=full, u=u, transition_first=tf),
                lgssm.kalman_rts(y, **omod, mask=full, u=u, transition_first=tf)):
        assert _rel(sm["mean"].numpy(), ref["mean"]) < 1e-10
        assert _rel(fl["mean"].numpy(), ref["filt_mean"]) < 1e-10
        assert _rel(np.broadcast_to(cs["Ss"][..., None], ref["cov"].shape), ref["cov"]) < 1e-10
        assert _rel(np.broadcast_to(cs["Sf"][..., None], ref["filt_cov"].shape), ref["filt_cov"]) < 1e-10
        for got in (sm["nle"].numpy(), fl["nle"].numpy()):
            assert np.all(np.abs(got - ref["neg_log_evidence"]) <= 1e-10 * np.maximum(1.0, np.abs(ref["neg_log_evidence"])))


@pytest.mark.parametrize("d,m,bkind", CPU_SHAPES)
def test_reference_matches_streaming_oracle(d, m, bkind):
    """Filtering with the prior one transition before the first datum, a per-chain prior mean and a carried prior
    covariance (the streaming chunk's prior) = the oracle's streaming filter."""
    mod = _cpu_model(d, m, bkind)
    y = simulate(mod, 25, 6, seed=7 * d + m)
    rng = np.random.default_rng(10 * d + m)
    mu0 = rng.standard_normal((d, 6))
    C = rng.standard_normal((d, d))
    mod2 = dict(mod, S0=np.asarray(2.0 * np.eye(d) + 0.2 * C @ C.T, np.float32).astype(np.float64))
    u = offset(d, 5).astype(np.float64)
    ref = lgssm.filter_streaming(y, **dict(mod2, m0=mu0.T.copy()), u=u)
    r = reference_sweep(mod2, torch.as_tensor(y), smooth=False, u=u, transition_first=True, mu0=torch.as_tensor(mu0))
    assert _rel(r["mean"].numpy(), ref["mean"]) < 1e-10
    assert _rel(np.broadcast_to(r["cov"][..., None], ref["cov"].shape), ref["cov"]) < 1e-10


# (T, batch) -> (tiles, tsplit, pre-pass slice lengths, evidence tiles, ev_slices, evidence slice lengths)
PINNED = {
    132: {(1000, 4096): (64, 5, [200], 128, 5, [200]),          # configs[2] on an H100 SXM
          (300, 16897): (265, 1, [300], 529, 1, [300]),
          (65, 64): (1, 65, [1], 2, 65, [1]),
          (257, 2000): (32, 9, [28, 29], 63, 9, [28, 29]),
          (128, 4225): (67, 4, [32], 133, 4, [32])},
    114: {(1000, 4096): (64, 4, [250], 128, 4, [250]),          # H100 PCIe
          (300, 16897): (265, 1, [300], 529, 1, [300]),
          (65, 64): (1, 65, [1], 2, 65, [1]),
          (257, 2000): (32, 8, [32, 33], 63, 8, [32, 33]),
          (128, 4225): (67, 4, [32], 133, 4, [32])},
}


@pytest.mark.parametrize("sm", sorted(PINNED))
def test_launch_geometry_is_pinned(sm):
    """The restated grid formulas at 132 and 114 SMs: a change to them in the kernels' launchers must show up here."""
    for (T, batch), want in PINNED[sm].items():
        g = launch_geometry(sm, T, batch)
        got = (g["tiles"], g["tsplit"], g["ky_steps"], g["ev_tiles"], g["ev_slices"], g["ev_steps"])
        assert got == want, (sm, T, batch, got)
    # the batches the slice-geometry test derives from the SM count
    assert launch_geometry(sm, 300, 128 * sm + 1)["tsplit"] == 1 and launch_geometry(sm, 300, 128 * sm + 1)["ev_slices"] == 1
    assert launch_geometry(sm, 300, 128 * sm - 64)["tsplit"] > 1
    b4 = batch_for(sm, 1 << 20, lambda g: g["ev_slices"] == 4)
    assert launch_geometry(sm, 4 * 33, b4)["ev_steps"] == [33]


# ====================================================================================== GPU: the native matrix
MATRIX_T = [1, 2, 3, 31, 32, 33, 64, 65, 257]
MAIN_B = 129                          # 2 wgmma tiles + 1 chain, 4 block / evidence tiles + 1 chain
EDGE_B = [1, 2, 31, 32, 33, 63, 64, 65, 96, 97]
OPTIONS = list(itertools.product((True, False), (False, True), (False, True)))      # smooth x evidence x transition_first
COV_MODES = ("chain", "shared", "none")


def impls(d):
    """(name, no_umma, large_seq): the default dispatch (wgmma sweep at d >= 16, block sweep at d = 8, gain tables by
    doubling), the FP32-pipe block sweep at d >= 16 and the sequential gain tables."""
    return [("default", 0, 0)] + ([("block", 1, 0)] if d >= 16 else []) + [("seq", 0, 1)]


def _run(ctx, y, mod, impl, *, smooth=True, evid=False, tf=False, cov_mode="none", u=None, **kw):
    ctx.set_option("no_umma", impl[1])
    ctx.set_option("large_seq", impl[2])
    return ctx.lgssm(y, **_kw(mod), u=u, smooth=smooth, want_cov=cov_mode != "none", want_evidence=evid,
                     cov_shared_out=cov_mode == "shared", transition_first=tf, **kw)


def _gate(cat, case, r, ref, cs, chains, *, smooth, evid, cov_mode, identical=True):
    gate_mean(CAT + cat, case, r["mean"], ref["mean"][..., chains])
    if evid:
        gate_nle(CAT + cat, case, r["neg_log_evidence"], ref["nle"][chains])
    else:
        assert r["neg_log_evidence"] is None
    if cov_mode != "none":
        gate_cov_steps(CAT + cat, case, r["cov"], cs["Ss"] if smooth else cs["Sf"], identical=identical)
    else:
        assert r["cov"] is None


@pytest.mark.gpu
@pytest.mark.parametrize("T", MATRIX_T)
@pytest.mark.parametrize("bkind", ["I", "dense"])
@pytest.mark.parametrize("d", NATIVE_D)
def test_native_matrix(ctx, d, bkind, T):
    """Smoothing / filtering x evidence x transition_first x covariance per chain / table / none, on every
    implementation at batch 129 (ragged last tile of every kernel), and on the default one again at a tile-edge batch
    (1, 2, 31-33, 63-65, 96, 97) over chains 3.., every chain gated.  Exact relations: evidence does not change the
    means; chain reversal and a sub-batch give the same per-chain bits; the table equals every chain's covariance; an
    all-zero offset is no offset."""
    mod = native_model(d, bkind)
    ti = MATRIX_T.index(T)
    y = torch.as_tensor(simulate(mod, T, MAIN_B, seed=97 * T + d + (bkind == "I")), device="cuda")
    cs = {tf: covariance_side(mod, T, None, tf) for tf in (False, True)}
    refs = {}
    for i, (smooth, evid, tf) in enumerate(OPTIONS):
        key = (smooth, tf)
        if key not in refs:
            refs[key] = reference_sweep(mod, y, smooth=smooth, transition_first=tf, cs=cs[tf])
        ref = refs[key]
        opt = f"d={d} B={bkind} T={T} {'smooth' if smooth else 'filter'} evid={int(evid)} tf={int(tf)}"
        cov_mode = COV_MODES[(i + ti) % 3]
        kw = dict(smooth=smooth, evid=evid, tf=tf)
        for impl in impls(d):
            case = f"{opt} {impl[0]} batch={MAIN_B} cov={cov_mode}"
            r = _run(ctx, y, mod, impl, cov_mode=cov_mode, **kw)
            _gate("matrix", case, r, ref, cs[tf], slice(None), smooth=smooth, evid=evid, cov_mode=cov_mode)
            # evidence runs a filter-mode sweep first; the means must not notice
            rn = _run(ctx, y, mod, impl, **dict(kw, evid=not evid))
            _eq(r["mean"], rn["mean"], "mean with / without evidence", case)
            # chain order reversed: every chain changes tile and row
            rr = _run(ctx, y.flip(-1).contiguous(), mod, impl, **kw)
            _eq(rr["mean"].flip(-1), r["mean"], "mean under chain reversal", case)
            if evid:
                _eq(rr["neg_log_evidence"].flip(-1), r["neg_log_evidence"], "nle under chain reversal", case)
            if impl[0] != "default":
                continue
            # a sub-batch at a tile edge, starting at chain 3: same per-chain bits as inside the batch of 129
            nb = EDGE_B[(i + 3 * ti) % len(EDGE_B)]
            ecov = COV_MODES[(i + ti + 1) % 3]
            ecase = f"{opt} {impl[0]} batch={nb} cov={ecov}"
            chains = slice(3, 3 + nb)
            re = _run(ctx, y[..., chains].contiguous(), mod, impl, cov_mode=ecov, **kw)
            _gate("matrix edge batch", ecase, re, ref, cs[tf], chains, smooth=smooth, evid=evid, cov_mode=ecov)
            _eq(re["mean"], r["mean"][..., chains], "sub-batch mean vs batch-129 mean", ecase)
            if ecov != "none" and cov_mode != "none":
                tab = lambda x: x[..., 0] if x.dim() == 4 else x
                _eq(tab(re["cov"]), tab(r["cov"]), "covariance table across batches / output modes", ecase)
            if i == 0:
                # an all-zero offset is dropped by the dispatcher: the same call as without one
                rz = _run(ctx, y, mod, impl, u=np.zeros(d, np.float32), cov_mode=cov_mode, **kw)
                _eq(rz["mean"], r["mean"], "mean with u = 0", case)
                _eq(rz["neg_log_evidence"], r["neg_log_evidence"], "nle with u = 0", case)
                _eq(rz["cov"], r["cov"], "cov with u = 0", case)


# ====================================================================================== GPU: slice geometry
def _slices_case(ctx, d, T, batch, cat, *, cov_mode="shared"):
    """Smoothing with evidence and filtering with evidence at one launch geometry, on the default sweep and (d >= 16)
    the block sweep, every chain and step gated."""
    mod = native_model(d, "I" if d % 32 == 0 else "dense")
    y = torch.as_tensor(simulate(mod, T, batch, seed=T + batch), device="cuda")
    cs = covariance_side(mod, T)
    for smooth in (True, False):
        ref = reference_sweep(mod, y, smooth=smooth, cs=cs)
        for impl in [i for i in impls(d) if i[0] != "seq"]:
            case = f"d={d} T={T} batch={batch} {'smooth' if smooth else 'filter'} {impl[0]}"
            r = _run(ctx, y, mod, impl, smooth=smooth, evid=True, cov_mode=cov_mode)
            _gate(cat, case, r, ref, cs, slice(None), smooth=smooth, evid=True, cov_mode=cov_mode)
            del r
        del ref
    torch.cuda.empty_cache()


@pytest.mark.gpu
def test_slices_one_step_each(ctx):
    """(a) the pre-pass and the evidence kernel with one time step per slice."""
    sm = sm_count()
    T, batch = 65, 64
    g = launch_geometry(sm, T, batch)
    assert g["ky_steps"] == [1] and g["ev_steps"] == [1], g
    _slices_case(ctx, 16, T, batch, "slices 1 step")


@pytest.mark.gpu
def test_slices_whole_series(ctx):
    """(b) tsplit = 1 and ev_slices = 1: one slice of 300 steps in both kernels (d = 16, 128 SM + 1 chains: one chain
    in the last wgmma and evidence tiles)."""
    sm = sm_count()
    T, batch = 300, 128 * sm + 1
    g = launch_geometry(sm, T, batch)
    assert g["tsplit"] == 1 and g["ev_slices"] == 1, g
    _slices_case(ctx, 16, T, batch, "slices whole series")


@pytest.mark.gpu
def test_slices_not_dividing_T(ctx):
    """(b) T = 257 (prime) cut into several slices of unequal length in both kernels (d = 32)."""
    sm = sm_count()
    T = 257
    batch = batch_for(sm, T, lambda g: 4 <= g["tsplit"] <= 16 and len(g["ky_steps"]) == 2 and len(g["ev_steps"]) == 2,
                      lo=1000)
    _slices_case(ctx, 32, T, batch, "slices uneven")


@pytest.mark.gpu
@pytest.mark.parametrize("steps", [31, 32, 33, 75])
def test_evidence_slices_around_the_flush(ctx, steps):
    """(c) evidence slices of 31, 32, 33 and 75 steps: the fp32 partial is flushed to fp64 every 32 steps of a slice.
    Four slices (batch from the SM count), T = 4 x steps; d = 8 (block sweep) and d = 16 (both sweeps)."""
    sm = sm_count()
    batch = batch_for(sm, 1 << 20, lambda g: g["ev_slices"] == 4)
    T = 4 * steps
    g = launch_geometry(sm, T, batch)
    assert g["ev_slices"] == 4 and g["ev_steps"] == [steps], g
    for d in (8, 16):
        _slices_case(ctx, d, T, batch, "evidence slices", cov_mode="none")


# ====================================================================================== GPU: configs[2] itself
@pytest.mark.gpu
def test_configs2_every_chain(ctx):
    """BASELINE configs[2]: d = 64, T = 1000, 4096 chains, the dense model, y = randn * 3.3 as bench.py draws it.
    Smoothing, filtering and smoothing with evidence (default dispatch: wgmma sweep), every chain and every step of the
    covariance table gated."""
    sm = sm_count()
    d, T, batch = 64, 1000, 4096
    g = launch_geometry(sm, T, batch)
    assert min(g["ky_steps"]) > 32 and min(g["ev_steps"]) > 32, g
    mod = f32_model(lgssm.dense_model(d))
    gen = torch.Generator(device="cuda").manual_seed(7)
    y = torch.randn(T, d, batch, device="cuda", generator=gen) * 3.3
    cs = covariance_side(mod, T)
    for smooth, evid in ((True, False), (False, False), (True, True)):
        case = f"configs[2] {'smooth' if smooth else 'filter'} evid={int(evid)} ({g['tsplit']} pre-pass / {g['ev_slices']} evidence slices)"
        r = ctx.lgssm(y, **_kw(mod), smooth=smooth, want_evidence=evid, cov_shared_out=True)
        ref = reference_sweep(mod, y, smooth=smooth, cs=cs)
        _gate("configs[2]", case, r, ref, cs, slice(None), smooth=smooth, evid=evid, cov_mode="shared")
        del r, ref
        torch.cuda.empty_cache()


@pytest.mark.gpu
def test_configs2_per_chain_covariance(ctx):
    """configs[2]'s per-chain covariance output (broadcast_cov_kernel) at T = 100 and 4096 chains (6.7 GB): every chain
    bit-identical to the table, the table gated at every step."""
    d, T, batch = 64, 100, 4096
    need = 4 * T * d * d * batch * 2 + (4 << 30)
    free, _ = torch.cuda.mem_get_info()
    if free < need:
        pytest.skip(f"needs {need / 2**30:.1f} GiB of free device memory, {free / 2**30:.1f} GiB free (shared device)")
    mod = f32_model(lgssm.dense_model(d))
    gen = torch.Generator(device="cuda").manual_seed(7)
    y = torch.randn(T, d, batch, device="cuda", generator=gen) * 3.3
    cs = covariance_side(mod, T)
    r = ctx.lgssm(y, **_kw(mod), smooth=True)
    ref = reference_sweep(mod, y, cs=cs)
    _gate("configs[2] per-chain cov", "d=64 T=100 batch=4096 smooth", r, ref, cs, slice(None), smooth=True, evid=False,
          cov_mode="chain")
    del r, ref
    torch.cuda.empty_cache()


# ====================================================================================== GPU: embedded shapes
@pytest.mark.gpu
@pytest.mark.parametrize("d,m", list(EMBEDDED))
def test_embedded_shapes(ctx, d, m):
    """General shapes on the large-state family (shared model): smoothing and filtering with evidence (the dummy
    observations' -(M - m) n_obs 1/2 log 2 pi correction), per-chain covariances and the table, and per-chain prior
    means through the streaming chunk, every chain gated."""
    mod = random_model(d, m, seed=7000 + 64 * d + m)
    T, nb = 45, 67
    y = torch.as_tensor(simulate(mod, T, nb, seed=d * 64 + m), device="cuda")
    cs = covariance_side(mod, T)
    for smooth, cov_mode in ((True, "chain"), (False, "shared"), (True, "shared"), (False, "chain")):
        case = f"({d}, {m}) -> {EMBEDDED[(d, m)]} {'smooth' if smooth else 'filter'} cov={cov_mode}"
        ref = reference_sweep(mod, y, smooth=smooth, cs=cs)
        r = _run(ctx, y, mod, ("default", 0, 0), smooth=smooth, evid=True, cov_mode=cov_mode)
        _gate("embedded", case, r, ref, cs, slice(None), smooth=smooth, evid=True, cov_mode=cov_mode)
    rng = np.random.default_rng(d + m)
    prev = torch.as_tensor(rng.standard_normal((d, nb)).astype(np.float32), device="cuda")
    C = rng.standard_normal((d, d))
    carry0 = np.asarray(2.0 * np.eye(d) + 0.2 * C @ C.T, np.float32)
    cmod = dict(mod, S0=carry0.astype(np.float64))
    ref = reference_sweep(cmod, y, smooth=False, transition_first=True, mu0=prev)
    cc = carry0.copy()
    r = ctx.lgssm_filter_chunk(y, mod["A"], mod["B"], mod["P"], mod["Q"], prev, cc, want_evidence=True)
    case = f"({d}, {m}) -> {EMBEDDED[(d, m)]} chunk, per-chain prior"
    gate_mean(CAT + "embedded", case, r["mean"], ref["mean"])
    gate_nle(CAT + "embedded", case, r["neg_log_evidence"], ref["nle"])
    gate_cov_steps(CAT + "embedded", case, r["cov"], ref["cov"])


# ====================================================================================== GPU: streaming chunks
@pytest.mark.gpu
@pytest.mark.parametrize("d", [16, 64])
@pytest.mark.parametrize("sweep", ["default", "block"])
def test_streaming_chunks(ctx, d, sweep):
    """`lgssm_filter_chunk` over uneven chunks (1, 30, 37, 32 steps): a random per-chain prior mean in the first chunk,
    each later chunk carrying the last filtered means and covariance.  Every chain against one reference filter over
    the whole series, the evidence summed over chunks, the carried covariance against the reference's."""
    mod = native_model(d, "dense")
    chunks = [1, 30, 37, 32]
    T, nb = sum(chunks), 97
    rng = np.random.default_rng(d)
    y = torch.as_tensor(simulate(mod, T, nb, seed=d + 1), device="cuda")
    prev = torch.as_tensor(rng.standard_normal((d, nb)).astype(np.float32), device="cuda")
    C = rng.standard_normal((d, d))
    carry = np.asarray(2.0 * np.eye(d) + 0.2 * C @ C.T, np.float32)
    cmod = dict(mod, S0=carry.astype(np.float64))
    cs = covariance_side(cmod, T, None, True)
    ref = reference_sweep(cmod, y, smooth=False, transition_first=True, mu0=prev, cs=cs)
    ctx.set_option("no_umma", int(sweep == "block"))
    means, nle, t0 = [], torch.zeros(nb, dtype=torch.float64, device="cuda"), 0
    for k, L in enumerate(chunks):
        case = f"d={d} {sweep} chunk {k} (steps {t0}..{t0 + L - 1})"
        r = ctx.lgssm_filter_chunk(y[t0:t0 + L].contiguous(), mod["A"], mod["B"], mod["P"], mod["Q"], prev, carry,
                                   want_evidence=True)
        gate_mean(CAT + "streaming", case, r["mean"], ref["mean"][t0:t0 + L])
        gate_cov_steps(CAT + "streaming", case, r["cov"], cs["Sf"][t0:t0 + L])
        np.testing.assert_array_equal(carry, r["cov"][-1, :, :, 0].cpu().numpy())       # the carry out
        e = _rel(carry, cs["Sf"][t0 + L - 1])
        _record(CAT + "streaming carry", e, case, -1)
        assert e < TOL_COV, f"{case}: carried covariance relative Frobenius {e:.3e}"
        means.append(r["mean"])
        nle += r["neg_log_evidence"].double()
        prev = r["mean"][-1].contiguous()
        t0 += L
    gate_mean(CAT + "streaming", f"d={d} {sweep} all chunks", torch.cat(means), ref["mean"])
    gate_nle(CAT + "streaming", f"d={d} {sweep} evidence summed over chunks", nle, ref["nle"])


# ====================================================================================== GPU: shared mask
@pytest.mark.gpu
@pytest.mark.parametrize("d", [8, 16])
def test_shared_mask(ctx, d):
    """A shared missing-data pattern at large d: expanded to a per-chain mask on the generic per-chain kernel, which
    needs the per-chain covariance output; the table output (or none) is refused with RXG_ERR_UNSUPPORTED."""
    from rxinfer_jl_b200 import _lib as L
    mod = native_model(d, "dense")
    T, nb = 65, 70
    tm = pattern(T)
    y_np = simulate(mod, T, nb, seed=d + 11)
    y_np[tm == 0] = 1.0e3                      # values at missing steps must not reach any output
    y = torch.as_tensor(y_np, device="cuda")
    cs = covariance_side(mod, T, tm)
    for smooth in (True, False):
        case = f"d={d} T={T} {'smooth' if smooth else 'filter'} shared mask"
        ref = reference_sweep(mod, y, smooth=smooth, cs=cs)
        r = ctx.lgssm(y, **_kw(mod), smooth=smooth, mask=tm, want_evidence=True)
        _gate("shared mask", case, r, ref, cs, slice(None), smooth=smooth, evid=True, cov_mode="chain", identical=False)
        for kw in (dict(cov_shared_out=True), dict(want_cov=False)):
            with pytest.raises(L.RxGaussError) as ei:
                ctx.lgssm(y, **_kw(mod), smooth=smooth, mask=tm, **kw)
            assert ei.value.code == L.RXG_ERR_UNSUPPORTED, (case, kw, ei.value.code)


# ====================================================================================== GPU: misaligned caller buffers
@pytest.mark.gpu
@pytest.mark.parametrize("d,sweep", [(8, "block"), (16, "default"), (16, "block")])
def test_misaligned_caller_buffers(ctx, d, sweep):
    """y, out_mean and out_cov at a 4-byte offset (not 8- or 16-byte aligned), odd and even batches: every output
    bit-identical to the call with aligned buffers."""
    mod = native_model(d, "dense")
    T = 37
    impl = (sweep, int(sweep == "block"), 0)

    def off4(*shape):
        n = int(np.prod(shape))
        t = torch.empty(n + 1, device="cuda")[1:].view(*shape)
        assert t.data_ptr() % 16 == 4 and t.is_contiguous()
        return t

    for nb in (70, 71):
        y = torch.as_tensor(simulate(mod, T, nb, seed=d + nb), device="cuda")
        y_mis = off4(T, d, nb).copy_(y)
        for smooth in (True, False):
            kw = dict(smooth=smooth, evid=True, tf=smooth, cov_mode="chain")
            case = f"d={d} {sweep} batch={nb} {'smooth' if smooth else 'filter'}"
            base = _run(ctx, y, mod, impl, **kw)
            for what, extra, yy in (("out_mean", dict(out_mean=off4(T, d, nb)), y),
                                    ("out_cov", dict(out_cov=off4(T, d, d, nb)), y),
                                    ("y", {}, y_mis)):
                r = _run(ctx, yy, mod, impl, **kw, **extra)
                _eq(r["mean"], base["mean"], f"mean with misaligned {what}", case)
                _eq(r["cov"], base["cov"], f"cov with misaligned {what}", case)
                _eq(r["neg_log_evidence"], base["neg_log_evidence"], f"nle with misaligned {what}", case)
            cs = covariance_side(mod, T, None, smooth)
            ref = reference_sweep(mod, y, smooth=smooth, transition_first=smooth, cs=cs)
            _gate("misaligned", case, base, ref, cs, slice(None), smooth=smooth, evid=True, cov_mode="chain")
