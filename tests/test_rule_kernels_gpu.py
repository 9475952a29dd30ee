"""The per-rule Gaussian and Wishart kernels (csrc/rxg_rules.cu for d in {1..6, 8} and the nine register-resident
(d_out, d_in) pairs, csrc/rxg_rules_large.cu for every other d <= 64) message by message and element by element,
against fp64 references built from the same fp32-rounded inputs, across the whole dispatch table.

Every message and every element is gated, with the strongest gate the rule admits:
  * bit-exact for the rules that round once per element (the sums of +, prod and MvNormalMeanCovariance, prod_wishart):
    the GPU must equal the same operation in numpy float32;
  * a rigorous forward-error bound |gpu - ref| <= gamma_k (|A||S||A|')_ij, gamma_k = k u / (1 - k u), for the products
    (*(:out), the Wishart lambda rule): the bound depends on the operands only, so cancellation cannot break it;
  * a condition-scaled ratio ||error|| / (u d kappa_2 ||operands||) under one constant per rule family for every output
    of a Cholesky inverse (conversions, marginal, *(:in), wishart_mean).
SPD inputs are Q diag(lambda) Q' with condition numbers swept over 1 ... 1e4 across one batch, messages scaled by 1e-3 / 1
/ 1e3 in turn; message counts sit on both sides of every CTA edge (128 messages per register-path CTA, 256 columns per
k_left_gemm CTA, 8 or 6 messages per k_cholinv_warp CTA).  The worst case of every (rule, path, d) is printed at the end.
"""
import numpy as np
import pytest
import torch

from oracle import rules as R
from oracle import vmp

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
REG_D = (1, 2, 3, 4, 5, 6, 8)                                           # RXG_DISPATCH_D / rules_small
LARGE_D = (7, 9, 15, 16, 17, 31, 32, 33, 57, 58, 59, 63, 64)            # k_left_gemm rows 16 | 17, 32 | 33; cholinv_warp
                                                                        # lanes with a second row at d > 32, 8 -> 6
                                                                        # messages per CTA between d = 58 and 59
REG_PAIRS = ((1, 1), (1, 2), (2, 2), (3, 3), (1, 4), (2, 4), (4, 4), (6, 6), (8, 8))     # RXG_DISPATCH_DODI / rules_small2
LARGE_PAIRS = ((2, 1), (4, 1), (4, 2), (1, 64), (64, 1), (17, 3), (3, 17), (33, 64), (64, 33), (5, 5), (7, 5))
SCALES = np.array([1.0, 1e3, 1e-3])

# condition-scaled gates, one per rule family: about 4x the worst ratio this module measured on one H100 80GB HBM3
# (700 W): 3.7 (conversions), 4.1 (marginal), 4.5 (*(:in)), 3.7 (wishart_mean), each at d = 1 or d_out = 1
RATIO_CONVERT = 15.0        # meancov_to_wmp / wmp_to_meancov
RATIO_MARGINAL = 16.0       # marginal_gaussian, k = 1 ... 8
RATIO_MUL_IN = 18.0         # *(:in)
RATIO_WISHART_MEAN = 15.0   # wishart_mean
TOL_MV_IID = 2.5e-7         # fused IID-Wishart VMP (fp64 inside), relative per data set: measured worst 5.8e-8

WORST = {}      # (rule, path, d) -> (worst ratio or error, message, n)


def _record(rule, d, value, msg, n):
    path = "reg" if (d in REG_D if isinstance(d, int) else d in REG_PAIRS) else "large"
    key = (rule, path, str(d))
    if key not in WORST or value > WORST[key][0]:
        WORST[key] = (float(value), int(msg), int(n))


@pytest.fixture(scope="module", autouse=True)
def _report_worst(request):
    yield
    if not WORST:
        return
    with request.config.pluginmanager.getplugin("capturemanager").global_and_fixture_disabled():
        print("\nper-rule kernels, worst message per (rule, path, d) (bit-exact rules: 0 = no mismatch; bounds: "
              "error / bound; condition-scaled: error / (u d kappa ||operands||)):")
        for key in sorted(WORST, key=lambda k: (k[0], k[1], len(k[2]), k[2])):
            v, msg, n = WORST[key]
            print(f"  {key[0]:<24s} {key[1]:<5s} d={key[2]:<8s} {v:.3e}  (message {msg} of {n})")


# ------------------------------------------------------------------------------------------------ data and layout
def r32(a):
    return np.asarray(a, dtype=np.float32).astype(np.float64)


def dev(a):
    """[n, ...] host -> [..., n] fp32 CUDA (the ABI's structure-of-arrays layout, message index innermost)."""
    return torch.as_tensor(np.ascontiguousarray(np.moveaxis(np.asarray(a, np.float32), 0, -1)), device="cuda")


def host(t):
    """[..., n] CUDA -> [n, ...] float32."""
    return np.ascontiguousarray(np.moveaxis(t.cpu().numpy(), -1, 0))


def spd(rng, n, d, kmax=1e4):
    """n SPD matrices Q diag(lambda) Q' (fp32-rounded) with condition numbers log-spaced over 1 ... kmax across the
    batch (shuffled), message i scaled by 1, 1e3, 1e-3 in turn."""
    Q = np.linalg.qr(rng.standard_normal((n, d, d)))[0]
    kap = np.geomspace(1.0, kmax, n) if n > 1 else np.array([kmax])
    rng.shuffle(kap)
    lam = kap[:, None] ** -np.linspace(0.0, 1.0, d)[None, :]
    S = SCALES[np.arange(n) % 3, None, None] * np.einsum("nij,nj,nkj->nik", Q, lam, Q)
    return r32(0.5 * (S + np.swapaxes(S, 1, 2)))


def vec(rng, n, d):
    return r32(rng.standard_normal((n, d)) * SCALES[np.arange(n) % 3, None])


def mat(rng, *shape):
    """A random fp32 matrix [..., r, c] whose rows are scaled by 1, 1e3, 1e-3 in turn."""
    r = shape[-2]
    return r32(rng.standard_normal(shape) * SCALES[np.arange(r) % 3, None])


def gamma(k):
    return k * U / (1.0 - k * U)


def ns_square(d):
    if d in REG_D:
        return (1, 7, 8, 9, 127, 128, 129, 255, 256, 257, 3001)
    if d <= 17:
        return (1, 7, 8, 9, 255, 256, 257, 3001)
    if d <= 58:
        return (1, 7, 8, 9, 257)
    return (1, 5, 6, 7, 13, 257)


def ns_pair(pair):
    if pair in REG_PAIRS:
        return (1, 7, 127, 128, 129, 257, 3001)
    return (1, 7, 8, 9, 255, 256, 257) if max(pair) <= 17 else (1, 6, 7, 9, 13, 257)


# ------------------------------------------------------------------------------------------------ gates
def _where(shape, flat):
    idx = np.unravel_index(int(flat), shape)
    return idx[0], tuple(int(j) for j in idx[1:])


def gate_exact(rule, d, got, want):
    """got == want element for element (both float32 [n, ...])."""
    got, want = np.asarray(got, np.float32), np.asarray(want, np.float32)
    assert got.shape == want.shape, (rule, got.shape, want.shape)
    bad = got != want
    n = got.shape[0]
    if bad.any():
        m, el = _where(got.shape, np.flatnonzero(bad)[0])
        pytest.fail(f"{rule}, d = {d}, n = {n}: {int(bad.sum())} elements differ from the fp32 reference; first at "
                    f"message {m}, element {el}: {got[m][el]!r} != {want[m][el]!r}")
    _record(rule, d, 0.0, n - 1, n)


def gate_bound(rule, d, got, ref, bound):
    """|got - ref| <= bound, element for element ([n, ...] each)."""
    err = np.abs(np.asarray(got, np.float64) - ref)
    ratio = np.where(bound > 0, err / np.where(bound > 0, bound, 1.0), np.where(err > 0, np.inf, 0.0))
    ratio[np.isnan(err)] = np.inf
    n = ratio.shape[0]
    w = int(np.argmax(ratio))
    m, el = _where(ratio.shape, w)
    _record(rule, d, ratio.flat[w], m, n)
    assert ratio.flat[w] <= 1.0, (f"{rule}, d = {d}, n = {n}: message {m}, element {el}: |{got[m][el]!r} - {ref[m][el]!r}| "
                                  f"= {err[m][el]:.3e} exceeds the forward-error bound {bound[m][el]:.3e}")


def gate_ratio(rule, d, err, scale, limit):
    """Per message err / scale <= limit ([n] each)."""
    ratio = np.where(np.isnan(err), np.inf, err / scale)
    n = ratio.shape[0]
    m = int(np.argmax(ratio))
    _record(rule, d, ratio[m], m, n)
    assert ratio[m] <= limit, f"{rule}, d = {d}, n = {n}: message {m}: condition-scaled error {ratio[m]:.3e} > {limit}"


def fro(a):
    return np.sqrt((np.asarray(a, np.float64) ** 2).reshape(a.shape[0], -1).sum(axis=1))


def bit_symmetric(rule, d, M):
    gate_exact(rule + " symmetry", d, M, np.swapaxes(M, 1, 2))


def status_ok(rule, d, st):
    st = st.cpu().numpy()
    bad = np.flatnonzero(st != 0)
    assert bad.size == 0, f"{rule}, d = {d}: status {st[bad[0]]} at SPD message {bad[0]}"


def apply(M, v):
    return np.einsum("nij,nj->ni", M, v)


# ------------------------------------------------------------------------------------------------ element-wise rules
@pytest.mark.parametrize("d", REG_D + LARGE_D)
def test_elementwise_rules_bit_exact(ctx, d):
    """MvNormalMeanCovariance(:out / :mu) with a shared Sigma (host array or device [d, d]) and a per-message one, the
    from-data rule, +(:out), +(:in) and prod in (xi, W): one fp32 rounding per element on both paths."""
    rng = np.random.default_rng(100 + d)
    for n in ns_square(d):
        mu, S, mu2, S2 = vec(rng, n, d), spd(rng, n, d), vec(rng, n, d), spd(rng, n, d)
        Sig = mat(rng, d, d)
        f = lambda a: a.astype(np.float32)
        Sig_dev = torch.as_tensor(f(Sig), device="cuda")
        Sig_n = np.broadcast_to(f(Sig), (n, d, d))
        for label, Sg, Sn in (("shared host", Sig, Sig_n), ("shared device", Sig_dev, Sig_n), ("per message", dev(S2), f(S2))):
            for which in ("out", "mean"):
                l0 = ctx.launches
                mo, So = ctx.rule_add_cov(dev(mu), dev(S), Sg, which)
                assert ctx.launches - l0 == (1 if d in REG_D else 2)       # one register kernel, or k_ew twice
                gate_exact(f"add_cov {which} mean", d, host(mo), f(mu))
                gate_exact(f"add_cov {which} {label}", d, host(So), f(S) + Sn)
            mo, So = ctx.rule_mean_from_data(dev(mu), Sg)
            gate_exact("from_data mean", d, host(mo), f(mu))
            gate_exact(f"from_data {label}", d, host(So), Sn)
        o, So = ctx.rule_add_out(dev(mu), dev(S), dev(mu2), dev(S2))
        gate_exact("add_out mean", d, host(o), f(mu) + f(mu2))
        gate_exact("add_out cov", d, host(So), f(S) + f(S2))
        o, So = ctx.rule_add_in(dev(mu), dev(S), dev(mu2), dev(S2))
        gate_exact("add_in mean", d, host(o), f(mu) - f(mu2))
        gate_exact("add_in cov", d, host(So), f(S) + f(S2))
        o, So = ctx.prod_gaussian(dev(mu), dev(S), dev(mu2), dev(S2))
        gate_exact("prod_gaussian xi", d, host(o), f(mu) + f(mu2))
        gate_exact("prod_gaussian W", d, host(So), f(S) + f(S2))


# ------------------------------------------------------------------------------------------------ *(:out)
@pytest.mark.parametrize("pair", REG_PAIRS + LARGE_PAIRS, ids=lambda p: f"{p[0]}x{p[1]}")
def test_mul_out_forward_error(ctx, rx, pair):
    """(A mu, A S A') within gamma_{d_in} |A||mu| and gamma_{2 d_in + 1} |A||S||A|', element by element; a shared A
    from the host and from the device, and a per-message A on every register shape (refused on the others)."""
    do, di = pair
    reg = pair in REG_PAIRS
    rng = np.random.default_rng(10 * do + di)
    for n in ns_pair(pair):
        mu, S = vec(rng, n, di), spd(rng, n, di)
        A = mat(rng, do, di)
        As = [("shared host", A, A[None]), ("shared device", torch.as_tensor(A.astype(np.float32), device="cuda"), A[None])]
        if reg:
            Am = mat(rng, n, do, di)
            As.append(("per message", dev(Am), Am))
        elif n == 7:
            with pytest.raises(rx.RxGaussError):
                ctx.rule_mul_out(dev(mat(rng, n, do, di)), dev(mu), dev(S))
        for label, Ag, An in As:
            mo, So = ctx.rule_mul_out(Ag, dev(mu), dev(S))
            mo, So = host(mo), host(So)
            Aa = np.abs(An)
            ref_mu, ref = R.multiplication_out(An, (mu, S))
            gate_bound(f"mul_out mean {label}", pair, mo, np.broadcast_to(ref_mu, (n, do)),
                       gamma(di) * np.einsum("nij,nj->ni", np.broadcast_to(Aa, (n, do, di)), np.abs(mu)))
            bound = gamma(2 * di + 1) * (Aa @ np.abs(S) @ np.swapaxes(Aa, 1, 2))
            gate_bound(f"mul_out cov {label}", pair, So, ref, np.broadcast_to(bound, ref.shape))
            if reg:
                bit_symmetric("mul_out cov", pair, So)
            else:
                gate_bound("mul_out cov symmetry", pair, So, np.swapaxes(So, 1, 2).astype(np.float64),
                           2 * np.broadcast_to(bound, ref.shape))


# ------------------------------------------------------------------------------------------------ *(:in)
@pytest.mark.parametrize("pair", REG_PAIRS + LARGE_PAIRS, ids=lambda p: f"{p[0]}x{p[1]}")
def test_mul_in_condition_scaled(ctx, pair):
    """(A' W mu, A' W A), W = cholinv(S_out), against fp64, scaled by u d_out kappa(S_out) and the operands' norms;
    status 0 for every SPD message; bit-symmetric on the register path.  On the large path the product half is gated
    rigorously against the fp32 W and W mu of k_cholinv_warp when meancov_to_wmp at d_out makes the same call (d_out not
    a register size); symmetric within twice that bound."""
    do, di = pair
    reg = pair in REG_PAIRS
    rng = np.random.default_rng(1000 + 10 * do + di)
    for n in ns_pair(pair):
        mu, S = vec(rng, n, do), spd(rng, n, do)
        A = mat(rng, do, di)
        As = [("shared host", A, A[None])]
        if reg:
            Am = mat(rng, n, do, di)
            As.append(("per message", dev(Am), Am))
        xo_ref, W = R.meancov_to_wmp(mu, S)
        kap = np.linalg.cond(S)
        for label, Ag, An in As:
            An = np.broadcast_to(An, (n, do, di))
            l0 = ctx.launches
            xi, Wi, st = ctx.rule_mul_in(Ag, dev(mu), dev(S))
            assert ctx.launches - l0 == (1 if reg else 4)                   # register kernel, or cholinv_warp + 3 left-GEMMs
            xi, Wi = host(xi), host(Wi)
            status_ok("mul_in", pair, st)
            At = np.swapaxes(An, 1, 2)
            nA = fro(An)
            den = U * do * kap * nA * fro(W)
            xi_ref, Wi_ref = R.multiplication_in((xo_ref, W), An)
            gate_ratio(f"mul_in W {label}", pair, fro(Wi - Wi_ref), den * nA, RATIO_MUL_IN)
            gate_ratio(f"mul_in xi {label}", pair, np.linalg.norm(xi - xi_ref, axis=1),
                       den * np.linalg.norm(mu, axis=1), RATIO_MUL_IN)
            if reg:
                bit_symmetric("mul_in W", pair, Wi)
                continue
            if do in REG_D:
                # the conversion at d_out runs the register kernel, not this k_cholinv_warp call: bound |W_fp32| by
                # |W| plus the conversion's gated error
                Wabs = np.abs(W) + (RATIO_CONVERT * U * do * kap * fro(W))[:, None, None]
            else:
                xo, Wh, _ = ctx.meancov_to_wmp(dev(mu), dev(S))
                xo, Wh = host(xo).astype(np.float64), host(Wh).astype(np.float64)
                Wabs = np.abs(Wh)
                gate_bound("mul_in W product", pair, Wi, At @ Wh @ An, gamma(2 * do + 1) * (np.abs(At) @ Wabs @ np.abs(An)))
                gate_bound("mul_in xi product", pair, xi, apply(At, xo), gamma(do) * apply(np.abs(At), np.abs(xo)))
            gate_bound("mul_in W symmetry", pair, Wi, np.swapaxes(Wi, 1, 2).astype(np.float64),
                       2 * gamma(2 * do + 1) * (np.abs(At) @ Wabs @ np.abs(An)))


# ------------------------------------------------------------------------------------------------ conversions, marginal
@pytest.mark.parametrize("d", REG_D + LARGE_D)
def test_conversions_condition_scaled(ctx, d):
    """meancov_to_wmp and wmp_to_meancov (one kernel): both outputs against fp64, status 0, bit-symmetric output."""
    rng = np.random.default_rng(2000 + d)
    for n in ns_square(d):
        for rule in ("meancov_to_wmp", "wmp_to_meancov"):
            v, M = vec(rng, n, d), spd(rng, n, d)
            l0 = ctx.launches
            vo, Mo, st = getattr(ctx, rule)(dev(v), dev(M))
            assert ctx.launches - l0 == 1
            vo, Mo = host(vo), host(Mo)
            status_ok(rule, d, st)
            v_ref, Mi = getattr(R, rule)(v, M)
            den = U * d * np.linalg.cond(M) * fro(Mi)
            gate_ratio(rule + " matrix", d, fro(Mo - Mi), den, RATIO_CONVERT)
            gate_ratio(rule + " vector", d, np.linalg.norm(vo - v_ref, axis=1), den * np.linalg.norm(v, axis=1),
                       RATIO_CONVERT)
            bit_symmetric(rule, d, Mo)


@pytest.mark.parametrize("d", (1, 2, 5, 8, 9, 17, 33, 59))
def test_marginal_every_k(ctx, d):
    """The product of k = 1 ... 8 (xi, W) messages and its mean_cov, on both paths."""
    rng = np.random.default_rng(3000 + d)
    for n in ((7, 129) if d in REG_D else (7, 9) if d < 59 else (5, 13)):
        for k in range(1, 9):
            xs, Ws = [vec(rng, n, d) for _ in range(k)], [spd(rng, n, d) for _ in range(k)]
            mu, S, st = ctx.marginal_gaussian([(dev(x), dev(W)) for x, W in zip(xs, Ws)])
            mu, S = host(mu), host(S)
            status_ok(f"marginal k={k}", d, st)
            mref, Sref = R.marginal_from_messages(list(zip(xs, Ws)))
            den = U * d * np.linalg.cond(sum(Ws)) * fro(Sref)
            gate_ratio("marginal cov", d, fro(S - Sref), den, RATIO_MARGINAL)
            gate_ratio("marginal mean", d, np.linalg.norm(mu - mref, axis=1),
                       den * sum(np.linalg.norm(x, axis=1) for x in xs), RATIO_MARGINAL)
            bit_symmetric("marginal cov", d, S)


# ------------------------------------------------------------------------------------------------ Wishart family
@pytest.mark.parametrize("d", REG_D)
def test_wishart_rules(ctx, d):
    """MvNormalMeanPrecision(:Lambda) within gamma_4 (|Vo| + |Vm| + |a - b||a - b|'), prod_wishart bit-exact,
    wishart_mean condition-scaled, every message."""
    rng = np.random.default_rng(4000 + d)
    for n in (1, 7, 127, 128, 129, 3001):
        mo, mm, Vo, Vm = vec(rng, n, d), vec(rng, n, d), spd(rng, n, d), spd(rng, n, d)
        df, iS = ctx.rule_mvnormal_precision_lambda(dev(mo), dev(Vo), dev(mm), dev(Vm))
        df, iS = host(df), host(iS)
        rdf, riS = R.mvnormal_meanprec_lambda((mo, Vo), (mm, Vm))
        gate_exact("lambda df", d, df, rdf)
        dl = mo - mm
        gate_bound("lambda inv_scale", d, iS, riS,
                   gamma(4) * (np.abs(Vo) + np.abs(Vm) + np.abs(dl)[:, :, None] * np.abs(dl)[:, None, :]))
        bit_symmetric("lambda inv_scale", d, iS)
        df1, df2 = r32(d + 1.0 + 20.0 * rng.random(n)), r32(d + 1.0 + 20.0 * rng.random(n))
        iS1, iS2 = spd(rng, n, d), spd(rng, n, d)
        f = lambda a: a.astype(np.float32)
        pdf, piS = ctx.prod_wishart(dev(df1), dev(iS1), dev(df2), dev(iS2))
        gate_exact("prod_wishart df", d, host(pdf), (f(df1) + f(df2)) - np.float32(d + 1))
        gate_exact("prod_wishart inv_scale", d, host(piS), f(iS1) + f(iS2))
        EL, st = ctx.wishart_mean(dev(df1), dev(iS1))
        EL = host(EL)
        status_ok("wishart_mean", d, st)
        ref = R.wishart_mean((df1, iS1))
        gate_ratio("wishart_mean", d, fro(EL - ref), U * d * np.linalg.cond(iS1) * fro(ref), RATIO_WISHART_MEAN)
        bit_symmetric("wishart_mean", d, EL)


@pytest.mark.parametrize("d", (7, 9))
def test_wishart_rules_refuse_shapes_without_a_kernel(ctx, rx, d):
    rng = np.random.default_rng(d)
    n = 9
    m, V, df = dev(vec(rng, n, d)), dev(spd(rng, n, d)), dev(r32(np.full(n, d + 2.0)))
    with pytest.raises(rx.RxGaussError):
        ctx.rule_mvnormal_precision_lambda(m, V, m, V)
    with pytest.raises(rx.RxGaussError):
        ctx.prod_wishart(df, V, df, V)
    with pytest.raises(rx.RxGaussError):
        ctx.wishart_mean(df, V)


@pytest.mark.parametrize("d", (1, 4, 5, 6))
def test_mv_iid_wishart_vmp_per_data_set(ctx, d):
    """The fused IID-Wishart VMP against oracle.vmp.mv_iid_wishart, every data set on its own (the initial E[P] rounded to
    fp32 for both, as the ABI receives it)."""
    rng = np.random.default_rng(5000 + d)
    N, batch = 150, 131
    ys = []
    for _ in range(batch):
        Lc = rng.standard_normal((d, d))
        ys.append(rng.random(d)[None, :] + rng.standard_normal((N, d)) @ np.linalg.cholesky(Lc @ Lc.T + 0.1 * np.eye(d)).T)
    y = r32(np.stack(ys, axis=-1))
    EP0 = r32(d * 1e12 * np.eye(d))
    ref = vmp.mv_iid_wishart(y, iterations=6, init_E_P=EP0)
    got = ctx.mv_iid_wishart_vmp(torch.as_tensor(y.astype(np.float32), device="cuda"), iterations=6, init_E_P=EP0)
    status_ok("mv_iid_wishart", d, got["status"])
    gate_exact("mv_iid_wishart df", d, got["df"].cpu().numpy(), ref["df"].astype(np.float32))
    for key in ("m_mean", "m_cov", "inv_scale"):
        g, r = np.moveaxis(got[key].cpu().numpy().astype(np.float64), -1, 0), np.moveaxis(ref[key], -1, 0)
        gate_ratio(f"mv_iid_wishart {key}", d, fro(g - r), fro(r), TOL_MV_IID)


def test_mv_iid_wishart_vmp_refuses_d7(ctx, rx):
    y = torch.zeros(10, 7, 3, device="cuda")
    with pytest.raises(rx.RxGaussError):
        ctx.mv_iid_wishart_vmp(y, iterations=2)


# ------------------------------------------------------------------------------------------------ isolation of bad messages
@pytest.mark.parametrize("d", (2, 4, 8, 9, 33, 59, 64))
def test_bad_messages_are_flagged_and_isolated(ctx, rx, d):
    """Indefinite and NaN messages next to CTA edges (127 | 128 of a register CTA; 5 | 6, 7 | 8 and 13 inside the
    8- or 6-message groups of k_cholinv_warp; the last message of a partial CTA): RXG_ERR_NOT_SPD exactly there, 0
    elsewhere, and every other message bit-identical to a run with those messages replaced by SPD ones."""
    rng = np.random.default_rng(6000 + d)
    n = 259
    bad = [0, 5, 6, 7, 8, 13, 127, 128, n - 1]
    mu, S = vec(rng, n, d), spd(rng, n, d)
    P, C = S.copy(), S.copy()
    C[bad] = spd(rng, len(bad), d)
    for j, i in enumerate(bad):
        if j % 3 == 0:                                                  # negated: the first pivot is negative
            P[i] = -P[i]
        elif j % 3 == 1:                                                # NaN in the lower triangle
            P[i, d - 1, 0] = P[i, 0, d - 1] = np.nan
        else:                                                           # one negative eigenvalue
            Q = np.linalg.qr(rng.standard_normal((d, d)))[0]
            P[i] = (Q * np.r_[np.ones(d - 1), -1.0]) @ Q.T
    A = mat(rng, d, d)
    want = np.zeros(n, np.int32)
    want[bad] = rx._lib.RXG_ERR_NOT_SPD
    ok = np.setdiff1d(np.arange(n), bad)
    runs = {
        "meancov_to_wmp": lambda M: ctx.meancov_to_wmp(dev(mu), dev(M)),
        "marginal k=2": lambda M: ctx.marginal_gaussian([(dev(mu), dev(M))] * 2),
        "mul_in": lambda M: ctx.rule_mul_in(A, dev(mu), dev(M)),
    }
    if d in REG_D:
        runs["wishart_mean"] = lambda M: ctx.wishart_mean(dev(r32(np.full(n, d + 3.0))), dev(M))
    for rule, run in runs.items():
        *outs_p, st_p = run(P)
        *outs_c, st_c = run(C)
        assert st_p.cpu().numpy().tolist() == want.tolist(), f"{rule}, d = {d}: status with bad messages"
        status_ok(rule + " (replaced)", d, st_c)
        for a, b in zip(outs_p, outs_c):
            gate_exact(f"isolation {rule}", d, host(a)[ok], host(b)[ok])


# ------------------------------------------------------------------------------------------------ wrappers
def test_shared_device_operands_match_host_operands(ctx):
    """A PointMass A or Sigma passed as a device [r, c] tensor is shared (not read as [r, c, n]): bit-identical to the
    host array, on both paths."""
    rng = np.random.default_rng(7)
    for d, n in ((4, 300), (6, 129), (16, 300), (33, 77)):
        mu, S = vec(rng, n, d), spd(rng, n, d)
        A, Sig = mat(rng, d, d), spd(rng, 1, d)[0]
        Ad, Sd = (torch.as_tensor(x.astype(np.float32), device="cuda") for x in (A, Sig))
        for f in (lambda M: ctx.rule_add_cov(dev(mu), dev(S), M, "out"), lambda M: ctx.rule_mean_from_data(dev(mu), M)):
            for a, b in zip(f(Sig), f(Sd)):
                gate_exact("device Sigma", d, host(b), host(a))
        for f in (lambda M: ctx.rule_mul_out(M, dev(mu), dev(S)), lambda M: ctx.rule_mul_in(M, dev(mu), dev(S))):
            for a, b in zip(f(A), f(Ad)):
                if a.dtype == torch.float32:
                    gate_exact("device A", d, host(b), host(a))


def test_call_rule_and_prod_accept_a_shared_covariance(ctx, rx):
    """MvNormalMeanCovariance documents Sigma as [d, d, n] or [d, d] shared by the batch: call_rule and prod expand the
    shared form, with results identical to the expanded covariance."""
    rng = np.random.default_rng(8)
    for d, n in ((3, 200), (17, 70)):
        mu, mu2, S2 = vec(rng, n, d), vec(rng, n, d), spd(rng, n, d)
        Sig = spd(rng, 1, d)[0]
        Sd = torch.as_tensor(Sig.astype(np.float32), device="cuda")
        Sx = Sd[:, :, None].expand(d, d, n).contiguous()
        shared, full = (rx.MvNormalMeanCovariance(dev(mu), s) for s in (Sd, Sx))
        other = rx.MvNormalMeanCovariance(dev(mu2), dev(S2))
        A = rx.PointMass(mat(rng, d, d))
        for got, want in ((rx.call_rule(ctx, "+", "out", m_in1=shared, m_in2=other),
                           rx.call_rule(ctx, "+", "out", m_in1=full, m_in2=other)),
                          (rx.call_rule(ctx, "*", "out", m_A=A, m_in=shared), rx.call_rule(ctx, "*", "out", m_A=A, m_in=full)),
                          (rx.call_rule(ctx, "MvNormalMeanCovariance", "out", **{"m_μ": shared, "q_Σ": rx.PointMass(Sig)}),
                           rx.call_rule(ctx, "MvNormalMeanCovariance", "out", **{"m_μ": full, "q_Σ": rx.PointMass(Sig)}))):
            gate_exact("call_rule shared cov mean", d, host(got.mu), host(want.mu))
            gate_exact("call_rule shared cov cov", d, host(got.Sigma), host(want.Sigma))
        got, want = rx.prod(ctx, shared, other), rx.prod(ctx, full, other)
        gate_exact("prod shared cov xi", d, host(got.xi), host(want.xi))
        gate_exact("prod shared cov W", d, host(got.W), host(want.W))
        got = rx.call_rule(ctx, "*", "in", m_out=shared, m_A=A)
        want = rx.call_rule(ctx, "*", "in", m_out=full, m_A=A)
        gate_exact("call_rule shared cov *(:in)", d, host(got.W), host(want.W))


def test_misshaped_operands_are_refused_before_any_launch(ctx, rx):
    """Every rule wrapper checks its operands against (d, n) before it launches.  Each operand here is at least as large
    as what a kernel would read, so a wrapper that did not check would give a wrong result, never an out-of-bounds
    access."""
    rng = np.random.default_rng(9)
    d, n = 4, 33
    mu, S, big = dev(vec(rng, n, d)), dev(spd(rng, n, d)), dev(spd(rng, n + 5, d))
    mu_big, df, df_big = dev(vec(rng, n + 5, d)), dev(r32(np.full(n, 7.0))), dev(r32(np.full(n + 5, 7.0)))
    A5 = mat(rng, d + 1, d + 1)
    cases = {
        "add_cov S": lambda: ctx.rule_add_cov(mu, big, np.eye(d)),
        "add_cov host Sigma": lambda: ctx.rule_add_cov(mu, S, A5),
        "add_cov per-message Sigma": lambda: ctx.rule_add_cov(mu, S, big),
        "from_data Sigma": lambda: ctx.rule_mean_from_data(mu, big),
        "mul_out S": lambda: ctx.rule_mul_out(np.eye(d), mu, big),
        "mul_out host A": lambda: ctx.rule_mul_out(A5, mu, S),
        "mul_out per-message A": lambda: ctx.rule_mul_out(big, mu, S),
        "mul_in S": lambda: ctx.rule_mul_in(np.eye(d), mu, big),
        "mul_in host A": lambda: ctx.rule_mul_in(A5, mu, S),
        "add_out second vector": lambda: ctx.rule_add_out(mu, S, mu_big, S),
        "add_in second matrix": lambda: ctx.rule_add_in(mu, S, mu, big),
        "prod first matrix": lambda: ctx.prod_gaussian(mu, big, mu, S),
        "conversion matrix": lambda: ctx.meancov_to_wmp(mu, big),
        "marginal second W": lambda: ctx.marginal_gaussian([(mu, S), (mu, big)]),
        "marginal second xi": lambda: ctx.marginal_gaussian([(mu, S), (mu_big, S)]),
        "lambda V_mu": lambda: ctx.rule_mvnormal_precision_lambda(mu, S, mu, big),
        "lambda m_mu": lambda: ctx.rule_mvnormal_precision_lambda(mu, S, mu_big, S),
        "prod_wishart df": lambda: ctx.prod_wishart(df, S, df_big, S),
        "prod_wishart second inverse scale": lambda: ctx.prod_wishart(df, S, df, big),
        "wishart_mean df": lambda: ctx.wishart_mean(df_big, S),
        "marginal no messages": lambda: ctx.marginal_gaussian([]),
    }
    for name, call in cases.items():
        l0 = ctx.launches
        with pytest.raises(ValueError):
            call()
        assert ctx.launches == l0, f"{name}: launched before refusing"
    with pytest.raises(rx.RxGaussError):
        ctx.marginal_gaussian([(mu, S)] * 9)
