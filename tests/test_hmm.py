"""Hidden Markov model, structured VMP q(s, s_0) q(A) q(B) (RxInfer test/models/statespace/hmm_tests.jl), on the CPU.

This module holds the fp64 reference the CUDA kernel (csrc/rxg_hmm.cuh) is gated against, as test_mixture.py does for the
Gaussian mixture:
  A ~ DirichletCollection(alpha_A0)   K x K, column j = p(s_t | s_{t-1} = j)
  B ~ DirichletCollection(alpha_B0)   M x K, column j = p(x_t | s_t = j)
  s_0 ~ Categorical(p0);  s[t] ~ DiscreteTransition(s[t-1], A);  x[t] ~ DiscreteTransition(s[t], B)
Either matrix may be known (a probability matrix) instead.  The chain is exact given exp(E[log A]), exp(E[log B]): one
scaled forward-backward sweep per iteration.  The checks here: the sweep against brute-force enumeration of every path,
the closed-form free energy against its dense definition under every schedule, the conjugate updates against the counts,
the monotone free energy, the column convention, the reference test's data and assertions, the kernel body compiled for the
host (tests/c/hmm_host_harness.cu), and the host-side argument handling."""
import ctypes
import itertools
import os
import shutil
import subprocess

import numpy as np
import pytest
from scipy.special import digamma, gammaln

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MISSING = 255
# Update orders tried against the reference's free-energy pin (DESIGN 3.18).  "sweep_update": the chain from the previous
# q(A), q(B), then both updated from the new q(s) (the kernel's order).  "b_lag": q(B) from the previous q(s) first (the
# initial q(s) at the first iteration), then the chain, then q(A).  "update_sweep": both from the previous q(s) first.
SCHEDULES = ("sweep_update", "b_lag", "update_sweep")


def elog_dir(alpha):
    """E[log A] of a DirichletCollection whose columns (axis 0 is the row) are independent Dirichlets."""
    return digamma(alpha) - digamma(alpha.sum(0, keepdims=True))


def kl_dir(a, a0):
    """sum over columns of KL(Dir(a[:, j]) || Dir(a0[:, j])); a [R, C, batch], a0 [R, C]."""
    a0 = a0[..., None]
    sa, sa0 = a.sum(0), a0.sum(0)
    return (gammaln(sa) - gammaln(a).sum(0) - gammaln(sa0) + gammaln(a0).sum(0)
            + ((a - a0) * (digamma(a) - digamma(sa)[None])).sum(0)).sum(0)


def emissions(x, Bt):
    """e[t, i, b] = Bt[x[t, b], i, b], 1 for a missing step.  x [T, batch], Bt [M, K, batch]."""
    T, nb = x.shape
    ok = x != MISSING
    xi = np.where(ok, x, 0).astype(np.int64)
    e = Bt[xi, :, np.arange(nb)[None, :]]                     # [T, batch, K]
    return np.where(ok[..., None], e, 1.0).transpose(0, 2, 1)


def forward_backward(x, p0, At, Bt, pairs=False):
    """Scaled forward-backward of every chain.  Returns q(s_t) gamma[T, K, b], q(s_0) gamma0[K, b], the transition counts
    xi[K, K, b] (sum_t q(s_t = i, s_{t-1} = j)), the emission counts nB[M, K, b], log Z~ [b] and, with ``pairs``, every
    q(s_{t-1}, s_t) as pair[T, K(next), K(prev), b]."""
    T, nb = x.shape
    K = At.shape[0]
    M = Bt.shape[0]
    e = emissions(x, Bt)
    alpha = np.zeros((T + 1, K, nb))
    alpha[0] = p0[:, None]
    logZ = np.zeros(nb)
    for t in range(1, T + 1):
        a = np.einsum("ijb,jb->ib", At, alpha[t - 1]) * e[t - 1]
        c = a.sum(0)
        alpha[t] = a / c
        logZ += np.log(c)
    beta = np.ones((K, nb))
    gamma = np.zeros((T + 1, K, nb))
    gamma[T] = alpha[T]
    xi = np.zeros((K, K, nb))
    pair = np.zeros((T, K, K, nb)) if pairs else None
    for t in range(T, 0, -1):
        w = e[t - 1] * beta
        p = At * w[:, None, :] * alpha[t - 1][None, :, :]
        p /= p.sum((0, 1))
        xi += p
        if pairs:
            pair[t - 1] = p
        gamma[t - 1] = p.sum(0)
        beta = np.einsum("ijb,ib->jb", At, w)
        beta /= (alpha[t - 1] * beta).sum(0)
    nB = np.zeros((M, K, nb))
    ok = x != MISSING
    for t in range(T):
        for b in np.nonzero(ok[t])[0]:
            nB[x[t, b], :, b] += gamma[t + 1, :, b]
    return dict(gamma=gamma[1:], gamma0=gamma[0], xi=xi, nB=nB, logZ=logZ, pair=pair)


def _side(prior, init, known, nb):
    if (known is None) == (prior is None):
        raise ValueError("exactly one of prior (with init) and known")
    if known is not None:
        k = np.asarray(known, np.float64)
        return None, None, np.repeat(k[..., None], nb, -1)
    return np.asarray(prior, np.float64), np.repeat(np.asarray(init, np.float64)[..., None], nb, -1), None


def closed_form_free_energy(st, logZ, A0, qA, A_used, B0, qB, B_used):
    """F = KL(q(A)||p(A)) + KL(q(B)||p(B)) - log Z~ + sum xi (E_used[log A] - E_new[log A]) + sum n_B (... B ...); the terms
    of a known matrix are omitted."""
    F = -logZ.copy()
    if A0 is not None:
        F += kl_dir(qA, A0) + (st["xi"] * (A_used - elog_dir(qA))).sum((0, 1))
    if B0 is not None:
        F += kl_dir(qB, B0) + (st["nB"] * (B_used - elog_dir(qB))).sum((0, 1))
    return F


def _xlogy(q, p):
    return np.where(q > 0, q * np.log(np.where(q > 0, p, 1.0)), 0.0)


def dense_free_energy(x, p0, st, A0, qA, Ak, B0, qB, Bk):
    """E_q[-log p(x, s, A, B)] - H[q(s, s_0)] - H[q(A)] - H[q(B)] from the pair marginals, term by term."""
    T, nb = x.shape
    pair = st["pair"]
    ElA = elog_dir(qA) if A0 is not None else None
    ElB = elog_dir(qB) if B0 is not None else None
    U = -_xlogy(st["gamma0"], p0[:, None]).sum(0)
    for t in range(T):
        U -= (pair[t] * ElA).sum((0, 1)) if A0 is not None else _xlogy(pair[t], Ak).sum((0, 1))
        ok = x[t] != MISSING
        xs = np.where(ok, x[t], 0)
        lb = (ElB if B0 is not None else None)
        for b in np.nonzero(ok)[0]:
            g = st["gamma"][t, :, b]
            U[b] -= (g * lb[xs[b], :, b]).sum() if B0 is not None else _xlogy(g, Bk[xs[b], :, b]).sum()
    H = np.zeros(nb)
    for t in range(T):
        H -= _xlogy(pair[t], pair[t]).sum((0, 1))
        if t < T - 1:
            H += _xlogy(st["gamma"][t], st["gamma"][t]).sum(0)
    for a0, q, El in ((A0, qA, ElA), (B0, qB, ElB)):
        if a0 is None:
            continue
        lnorm0 = (gammaln(a0.sum(0)) - gammaln(a0).sum(0)).sum()
        U -= lnorm0 + ((a0[..., None] - 1) * El).sum((0, 1))                                 # -E_q[log p(A)]
        H += -(gammaln(q.sum(0)) - gammaln(q).sum(0)).sum(0) - ((q - 1) * El).sum((0, 1))    # H[q(A)]
    return U - H


def hmm_vmp(x, p0, A_prior=None, A_init=None, A_known=None, B_prior=None, B_init=None, B_known=None, iterations=1,
            schedule="sweep_update", dense=False):
    """fp64 structured VMP of every chain.  x[T, batch] (symbols 0..M-1, 255 = missing).  Returns s_prob[T, K, b],
    s0_prob[K, b], A_alpha[K, K, b], B_alpha[M, K, b] (None when known), free_energy[its, b] and the KeepEach histories
    hist_s[its, T, K, b], hist_A, hist_B; with ``dense`` also free_energy_dense (the definition, term by term)."""
    x = np.asarray(x)
    T, nb = x.shape
    p0 = np.asarray(p0, np.float64)
    K = p0.shape[0]
    A0, qA, Ak = _side(A_prior, A_init, A_known, nb)
    B0, qB, Bk = _side(B_prior, B_init, B_known, nb)
    M = (B0 if B0 is not None else Bk).shape[0]
    uniform = dict(xi=np.full((K, K, nb), T / K ** 2), nB=np.zeros((M, K, nb)))   # statistics of the vague initial q(s)
    ok = x != MISSING
    for t in range(T):
        for b in np.nonzero(ok[t])[0]:
            uniform["nB"][x[t, b], :, b] += 1.0 / K
    prev = uniform
    out = {k: [] for k in ("free_energy", "free_energy_dense", "hist_s", "hist_A", "hist_B")}
    for _ in range(iterations):
        if schedule in ("b_lag", "update_sweep") and B0 is not None:
            qB = B0[..., None] + prev["nB"]
        if schedule == "update_sweep" and A0 is not None:
            qA = A0[..., None] + prev["xi"]
        A_used = elog_dir(qA) if A0 is not None else None
        B_used = elog_dir(qB) if B0 is not None else None
        At = np.exp(A_used) if A0 is not None else Ak
        Bt = np.exp(B_used) if B0 is not None else Bk
        st = forward_backward(x, p0, At, Bt, pairs=dense)
        if schedule in ("sweep_update", "b_lag") and A0 is not None:
            qA = A0[..., None] + st["xi"]
        if schedule == "sweep_update" and B0 is not None:
            qB = B0[..., None] + st["nB"]
        prev = st
        out["free_energy"].append(closed_form_free_energy(st, st["logZ"], A0, qA, A_used, B0, qB, B_used))
        if dense:
            out["free_energy_dense"].append(dense_free_energy(x, p0, st, A0, qA, Ak, B0, qB, Bk))
        out["hist_s"].append(st["gamma"])
        out["hist_A"].append(qA)
        out["hist_B"].append(qB)
    r = dict(s_prob=st["gamma"], s0_prob=st["gamma0"], A_alpha=qA, B_alpha=qB, xi=st["xi"], nB=st["nB"],
             free_energy=np.stack(out["free_energy"]), hist_s=np.stack(out["hist_s"]),
             hist_A=np.stack(out["hist_A"]) if A0 is not None else None,
             hist_B=np.stack(out["hist_B"]) if B0 is not None else None)
    if dense:
        r["free_energy_dense"] = np.stack(out["free_energy_dense"])
    return r


# --------------------------------------------------------------------------- the reference test's data and model
def _inverse_cdf_draw(rng, p):
    """rand(rng, Categorical(p)), one draw: Distributions' DiscreteNonParametric sampler, a linear search of the running
    sum against one rand(rng) (1-based)."""
    u = rng.rand()
    cp, i = p[0], 0
    while cp <= u and i < len(p) - 1:
        i += 1
        cp += p[i]
    return i + 1


def reference_data(seed=123, n=100):
    """hmm_tests.jl:54-82: StableRNG(123); s[t] = rand(Categorical(A s[t-1])), x[t] = rand(Categorical(B s[t])), s_0 = e_1.
    Returns the 0-based symbols x[n] and states s[n]."""
    from oracle.julia_rng import StableRNG
    rng = StableRNG(seed)
    A = np.array([[0.9, 0.0, 0.1], [0.1, 0.9, 0.0], [0.0, 0.1, 0.9]])
    B = np.array([[0.9, 0.05, 0.05], [0.05, 0.9, 0.05], [0.05, 0.05, 0.9]])
    s_prev = np.array([1.0, 0.0, 0.0])
    xs, ss = [], []
    for _ in range(n):
        a = A @ s_prev
        s = _inverse_cdf_draw(rng, list(a / a.sum())) - 1
        b = B[:, s]
        xo = _inverse_cdf_draw(rng, list(b / b.sum())) - 1
        ss.append(s); xs.append(xo)
        s_prev = np.eye(3)[s]
    return np.array(xs, np.uint8), np.array(ss)


def reference_model():
    """hmm_tests.jl:8-30: priors, p0 and the vague initial q(A), q(B)."""
    return dict(p0=np.full(3, 1.0 / 3.0), A_prior=np.ones((3, 3)), A_init=np.ones((3, 3)),
                B_prior=np.array([[10.0, 1.0, 1.0], [1.0, 10.0, 1.0], [1.0, 1.0, 10.0]]), B_init=np.ones((3, 3)))


def f32(a):
    return None if a is None else np.asarray(a, np.float32).astype(np.float64)


def random_problem(K, M, T, nb, seed, learn_A=True, learn_B=True, p_missing=0.0, sharp=False):
    """Non-symmetric priors and initial marginals (they pin the column convention), or known matrices; data sampled from
    a random HMM with some missing steps."""
    rng = np.random.default_rng(seed)
    A = rng.dirichlet(np.full(K, 0.5), K).T                      # columns are the conditionals
    if sharp:
        A = 0.999 * np.eye(K) + 0.001 * A
    B = rng.dirichlet(np.full(M, 0.7), K).T
    p0 = rng.dirichlet(np.ones(K))
    x = np.zeros((T, nb), np.uint8)
    for b in range(nb):
        s = rng.choice(K, p=p0)
        for t in range(T):
            s = rng.choice(K, p=A[:, s])
            x[t, b] = rng.choice(M, p=B[:, s])
    x[rng.random((T, nb)) < p_missing] = MISSING
    kw = dict(p0=p0)
    if learn_A:
        kw.update(A_prior=rng.uniform(0.3, 3.0, (K, K)), A_init=rng.uniform(0.5, 4.0, (K, K)))
    else:
        kw.update(A_known=A)
    if learn_B:
        kw.update(B_prior=rng.uniform(0.3, 3.0, (M, K)), B_init=rng.uniform(0.5, 4.0, (M, K)))
    else:
        kw.update(B_known=B)
    return x, kw


def brute_force(x, p0, A, B):
    """q(s_t), q(s_{t-1}, s_t) and log p(x) by summing over all K^(T+1) paths of one chain."""
    T, K = len(x), len(p0)
    lp, paths = [], list(itertools.product(range(K), repeat=T + 1))
    for s in paths:
        v = np.log(p0[s[0]])
        for t in range(T):
            v += np.log(A[s[t + 1], s[t]])
            if x[t] != MISSING:
                v += np.log(B[x[t], s[t + 1]])
        lp.append(v)
    lp = np.array(lp)
    logp = np.log(np.exp(lp - lp.max()).sum()) + lp.max()
    w = np.exp(lp - logp)
    gamma, pair = np.zeros((T, K)), np.zeros((T, K, K))
    for s, wi in zip(paths, w):
        for t in range(T):
            gamma[t, s[t + 1]] += wi
            pair[t, s[t + 1], s[t]] += wi
    return gamma, pair, logp


@pytest.mark.parametrize("T,p_missing", [(1, 0.0), (4, 0.0), (6, 0.0), (6, 0.4)])
def test_known_matrices_equal_brute_force_enumeration(T, p_missing):
    x, kw = random_problem(3, 4, T, 3, seed=T + int(10 * p_missing), learn_A=False, learn_B=False, p_missing=p_missing)
    if p_missing:
        x[2, 0] = MISSING
    r = hmm_vmp(x, **kw, iterations=1, dense=True)
    st = forward_backward(x, kw["p0"], np.repeat(kw["A_known"][..., None], 3, -1), np.repeat(kw["B_known"][..., None], 3, -1),
                          pairs=True)
    for b in range(3):
        g, pair, logp = brute_force(x[:, b], kw["p0"], kw["A_known"], kw["B_known"])
        assert np.abs(r["s_prob"][:, :, b] - g).max() < 1e-12
        assert np.abs(st["pair"][..., b] - pair).max() < 1e-12
        assert abs(r["free_energy"][0, b] + logp) < 1e-10                 # F = -log p(x) with both matrices known
        assert abs(r["free_energy_dense"][0, b] + logp) < 1e-10


@pytest.mark.parametrize("schedule", SCHEDULES)
@pytest.mark.parametrize("learn", [(True, True), (True, False), (False, True)])
def test_closed_form_free_energy_equals_the_definition(schedule, learn):
    x, kw = random_problem(3, 5, 12, 4, seed=5, learn_A=learn[0], learn_B=learn[1], p_missing=0.2)
    r = hmm_vmp(x, **kw, iterations=4, schedule=schedule, dense=True)
    assert np.abs(r["free_energy"] - r["free_energy_dense"]).max() < 1e-10


def test_every_update_is_the_count_based_conjugate_update():
    x, kw = random_problem(4, 3, 15, 3, seed=8, p_missing=0.25)
    r1 = hmm_vmp(x, **kw, iterations=1, dense=True)
    nb = x.shape[1]
    At = np.exp(elog_dir(np.repeat(kw["A_init"][..., None], nb, -1)))
    Bt = np.exp(elog_dir(np.repeat(kw["B_init"][..., None], nb, -1)))
    st = forward_backward(x, kw["p0"], At, Bt, pairs=True)
    xi = st["pair"].sum(0)
    nB = np.zeros_like(r1["B_alpha"])
    for t in range(x.shape[0]):
        for b in range(nb):
            if x[t, b] != MISSING:
                nB[x[t, b], :, b] += st["pair"][t, :, :, b].sum(1)
    assert np.abs(r1["A_alpha"] - (kw["A_prior"][..., None] + xi)).max() < 1e-12
    assert np.abs(r1["B_alpha"] - (kw["B_prior"][..., None] + nB)).max() < 1e-12
    assert np.abs(r1["s_prob"] - st["pair"].sum(2)).max() < 1e-12


@pytest.mark.parametrize("schedule", SCHEDULES)
def test_free_energy_never_increases(schedule):
    for seed in range(4):
        x, kw = random_problem(3 + seed, 4, 40, 3, seed=seed, p_missing=0.1)
        fe = hmm_vmp(x, **kw, iterations=15, schedule=schedule)["free_energy"]
        assert np.all(np.diff(fe, axis=0) < 1e-9), (schedule, seed)


def test_non_symmetric_prior_pins_the_column_convention():
    """Columns are the conditionals: with A known to move state j to state (j + 1) mod K, the state after an observed
    state is its successor; the transposed reading would put it at the predecessor."""
    K, M = 3, 3
    A = np.roll(np.eye(K), 1, axis=0)                             # A[(j + 1) % K, j] = 1
    B = 0.98 * np.eye(M) + 0.01
    B /= B.sum(0)
    x = np.array([[0], [MISSING], [MISSING]], np.uint8)
    r = hmm_vmp(x, np.full(K, 1 / K), A_known=A, B_known=B)
    assert r["s_prob"][1, 1, 0] > 0.9 and r["s_prob"][2, 2, 0] > 0.9
    # and the learned counts land in the column of the conditioning state: with a non-symmetric prior and p0 = e_1, the
    # column sums of the A counts are the occupancies of s_0 .. s_{T-1} and the row sums those of s_1 .. s_T; the row sums
    # of the B counts are the number of times each symbol was observed.  The transposed reading swaps each pair.
    count_identities(lambda x, kw, its: hmm_vmp(x, **kw, iterations=its))


def count_identities(run):
    """The identities above, for ``run(x, kw, iterations)`` returning q(s_t), q(s_0) and the Dirichlet parameters."""
    x, kw = random_problem(3, 4, 60, 2, seed=3, p_missing=0.2)
    kw["p0"] = np.array([1.0, 0.0, 0.0])
    kw["A_prior"] = np.array([[5.0, 0.1, 0.1], [0.1, 0.1, 5.0], [0.1, 5.0, 0.1]])
    r = run(x, kw, 3)
    nA = np.asarray(r["A_alpha"], np.float64) - kw["A_prior"][..., None]
    nB = np.asarray(r["B_alpha"], np.float64) - kw["B_prior"][..., None]
    g, g0 = np.asarray(r["s_prob"], np.float64), np.asarray(r["s0_prob"], np.float64)
    occ_prev = g0 + g[:-1].sum(0)                                # [K, b]
    occ_next = g.sum(0)
    assert np.abs(nA.sum(0) - occ_prev).max() < 1e-4 and np.abs(nA.sum(1) - occ_next).max() < 1e-4
    assert np.abs(occ_prev - occ_next).max() > 0.5               # the pairs differ, so a transposed A would fail above
    seen = np.stack([(x == m).sum(0) for m in range(4)])         # [M, b]
    assert np.abs(nB.sum(1) - seen).max() < 1e-4
    assert np.abs(nB.sum(0) - np.where(x[:, None, :] != MISSING, g, 0).sum(0)).max() < 1e-4


# --------------------------------------------------------------------------- the reference test on the oracle
PIN = 60.614480654


def reference_assertions(hist_s, hist_A, hist_B, fe, iters=20, n=100):
    """hmm_tests.jl:92-96 on one chain."""
    assert len(hist_s) == iters and all(len(s) == n for s in hist_s)
    assert len(hist_A) == iters and len(hist_B) == iters
    d = np.diff(fe)
    assert len(fe) == iters and np.all(d[np.abs(d) > 1e-3] < 0)
    assert abs(fe[-1] - PIN) < 0.01


def test_reference_data_and_assertions_on_the_oracle():
    x, s = reference_data()
    assert x.shape == (100,) and set(np.unique(x)) <= {0, 1, 2}
    assert np.mean(x == s) > 0.8                                  # B is 0.9 on the diagonal
    for schedule in SCHEDULES:                                    # every order tried meets the pin's 0.01 (DESIGN 3.18)
        r = hmm_vmp(x[:, None], **reference_model(), iterations=20, schedule=schedule)
        reference_assertions(r["hist_s"][..., 0], r["hist_A"], r["hist_B"], r["free_energy"][:, 0])
    assert abs(hmm_vmp(x[:, None], **reference_model(), iterations=20)["free_energy"][-1, 0] - 60.61529361) < 1e-6


# --------------------------------------------------------------------------- the kernel body on the host
def host_params(K, M, p0, A_prior=None, A_init=None, A_known=None, B_prior=None, B_init=None, B_known=None):
    """The fp64 constant block of rxg_hmm_vmp_f32 (rxg::hmm::off_*) from fp32-rounded inputs."""
    A = A_known if A_known is not None else A_prior
    Ai = A_init if A_known is None else np.zeros((K, K))
    B = B_known if B_known is not None else B_prior
    Bi = B_init if B_known is None else np.zeros((M, K))
    return np.concatenate([f32(v).reshape(-1) for v in (p0, A, Ai, B, Bi)])


def _host_harness():
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    so = os.path.join(ROOT, "tests", "c", "_hmm_host.so")
    src = os.path.join(ROOT, "tests", "c", "hmm_host_harness.cu")
    hdr = os.path.join(ROOT, "rxinfer.jl_b200", "csrc", "rxg_hmm.cuh")
    if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(src), os.path.getmtime(hdr)):
        subprocess.run([nvcc, "-O2", "-Wno-deprecated-gpu-targets", "-shared", "-Xcompiler", "-fPIC", "-o", so, src], check=True)
    return ctypes.CDLL(so)


def run_host(lib, x, kw, iterations):
    T, nb = x.shape
    K = len(kw["p0"])
    la, lb = "A_prior" in kw, "B_prior" in kw
    M = (kw["B_prior"] if lb else kw["B_known"]).shape[0]
    prm = host_params(K, M, **kw)
    z = lambda *s: np.zeros(s, np.float32)
    out = dict(s_prob=z(T, K, nb), s0_prob=z(K, nb), A_alpha=z(K, K, nb), B_alpha=z(M, K, nb),
               free_energy=np.zeros((iterations, nb)), hist_s=z(iterations, T, K, nb), hist_A=z(iterations, K, K, nb),
               hist_B=z(iterations, M, K, nb), status=np.zeros(nb, np.int32))
    P = lambda a: a.ctypes.data_as(ctypes.c_void_p)
    xx = np.ascontiguousarray(x, np.uint8)
    rc = lib.hmm_host_run(K, M, T, ctypes.c_longlong(nb), iterations, int(la), int(lb), P(prm), P(xx), P(out["s_prob"]),
                          P(out["s0_prob"]), P(out["A_alpha"]), P(out["B_alpha"]), P(out["free_energy"]), P(out["hist_s"]),
                          P(out["hist_A"]), P(out["hist_B"]), P(out["status"]))
    assert rc == 0
    return out


def per_chain_rel(got, want):
    ax = tuple(range(got.ndim - 1))
    return (np.sqrt(((got - want) ** 2).sum(ax)) / np.maximum(np.sqrt((want ** 2).sum(ax)), 1e-30)).max()


def gate(case, r, ref, chains=None, tol_mean=1e-5, tol_s=1e-3, fe_tol=1e-5):
    """Per chain: alpha_A, alpha_B (and their histories) at tol_mean relative L2, q(s) at tol_s absolute, the free energy
    at fe_tol relative to max(|F|, 1) and non-increasing."""
    sel = (lambda v: v[..., chains]) if chains is not None else (lambda v: v)
    assert np.all(sel(np.asarray(r["status"])) == 0), case
    for k in ("A_alpha", "B_alpha", "hist_A", "hist_B"):
        if ref[k] is not None:
            e = per_chain_rel(sel(np.asarray(r[k], np.float64)), sel(ref[k]))
            assert e < tol_mean, f"{case}: {k} {e:.3g}"
    for k in ("s_prob", "s0_prob", "hist_s"):
        e = np.abs(sel(np.asarray(r[k], np.float64)) - sel(ref[k])).max()
        assert e < tol_s, f"{case}: {k} {e:.3g}"
    fe, fr = sel(np.asarray(r["free_energy"])), sel(ref["free_energy"])
    e = (np.abs(fe - fr) / np.maximum(np.abs(fr), 1.0)).max()
    assert e < fe_tol, f"{case}: free energy {e:.3g}"
    assert np.all(np.diff(fe, axis=0) <= 2 * fe_tol * np.maximum(np.abs(fe[:-1]), 1.0)), case


def reference_on_f32(x, kw, iterations):
    return hmm_vmp(x, **{k: f32(v) for k, v in kw.items()}, iterations=iterations)


@pytest.mark.parametrize("K", [2, 3, 4, 5, 6, 7, 8])
def test_kernel_body_on_the_host_matches_the_reference(K):
    lib = _host_harness()
    for M in (2, 5, 16):
        for la, lb in ((True, True), (False, True), (True, False), (False, False)):
            T, its = (37, 6) if la or lb else (37, 1)
            x, kw = random_problem(K, M, T, 3, seed=100 * K + M + 10 * la + 20 * lb, learn_A=la, learn_B=lb, p_missing=0.15)
            r = run_host(lib, x, kw, its)
            gate(f"K={K} M={M} learn A={la} B={lb}", r, reference_on_f32(x, kw, its), tol_s=1e-5)


def test_kernel_body_on_the_host_keeps_the_column_convention():
    lib = _host_harness()
    count_identities(lambda x, kw, its: run_host(lib, x, kw, its))


def test_kernel_body_on_the_host_reproduces_the_reference_pin():
    lib = _host_harness()
    x, _ = reference_data()
    r = run_host(lib, x[:, None], reference_model(), 20)
    reference_assertions(r["hist_s"][..., 0], r["hist_A"], r["hist_B"], r["free_energy"][:, 0])


def test_kernel_body_on_the_host_flags_bad_chains_only():
    """A symbol >= M (not 255) flags its chain RXG_ERR_BAD_ARG and is read as missing; a step impossible under known
    matrices (a zero normaliser) flags RXG_ERR_NAN; the neighbours keep their results."""
    lib = _host_harness()
    x, kw = random_problem(3, 4, 20, 4, seed=9)
    x[5, 1] = 7
    r = run_host(lib, x, kw, 3)
    assert list(r["status"]) == [0, 1, 0, 0]
    xm = x.copy(); xm[5, 1] = MISSING
    ref = reference_on_f32(xm, kw, 3)
    gate("bad symbol", r, ref, chains=[0, 2, 3], tol_s=1e-5)
    assert per_chain_rel(r["A_alpha"][..., [1]].astype(np.float64), ref["A_alpha"][..., [1]]) < 1e-5   # read as missing
    K, M = 3, 3
    A = np.roll(np.eye(K), 1, axis=0)
    x = np.zeros((4, 3), np.uint8)
    x[:, 1] = [1, 2, 1, 0]                                       # state 1 then 2 then back to 1: impossible
    x[:, 0] = [1, 2, 0, 1]
    x[:, 2] = [MISSING, 2, 0, MISSING]
    kwk = dict(p0=np.array([1.0, 0.0, 0.0]), A_known=A, B_known=np.eye(M))
    r = run_host(lib, x, kwk, 1)
    assert list(r["status"]) == [0, 5, 0]
    ref = reference_on_f32(x[:, [0, 2]], kwk, 1)
    assert np.abs(r["s_prob"][..., [0, 2]] - ref["s_prob"]).max() < 1e-6
    assert np.abs(r["free_energy"][:, [0, 2]] - ref["free_energy"]).max() < 1e-6


# --------------------------------------------------------------------------- host-side argument handling
def test_one_hot_conversion_and_argument_handling(rx):
    import torch
    from rxinfer_jl_b200 import Categorical, DirichletCollection, PointMass, vague
    from rxinfer_jl_b200.inference import hidden_markov_model, hmm_symbols, hmm_arguments, HMMConstraints
    x, _ = reference_data()
    oh = torch.zeros(100, 3, 2)
    oh[torch.arange(100), torch.as_tensor(x, dtype=torch.long), 0] = 1.0
    oh[:, :, 1] = oh[:, :, 0]
    oh[7, :, 1] = float("nan")                                    # a missing step
    sym = hmm_symbols(oh, 3)
    assert sym.dtype == torch.uint8 and sym.shape == (100, 2)
    assert np.array_equal(sym[:, 0].numpy(), x) and int(sym[7, 1]) == MISSING
    assert torch.equal(hmm_symbols(sym, 3), sym)
    soft = oh.clone(); soft[3, :, 0] = torch.tensor([0.5, 0.5, 0.0])
    with pytest.raises(ValueError, match="one-hot"):
        hmm_symbols(soft, 3)
    with pytest.raises(ValueError, match="M = 4"):
        hmm_symbols(oh, 4)
    assert np.allclose(vague(DirichletCollection, (3, 2)).alpha, np.ones((3, 2)))
    assert np.allclose(vague(Categorical, 4).p, np.full(4, 0.25))
    assert np.allclose(DirichletCollection(np.array([[1.0, 3.0], [3.0, 1.0]])).mean(), [[0.25, 0.75], [0.75, 0.25]])
    model = hidden_markov_model(p0=np.full(3, 1 / 3), A=DirichletCollection(np.ones((3, 3))),
                                B=DirichletCollection(np.eye(3) * 9 + 1))
    init = {"A": vague(DirichletCollection, (3, 3)), "B": vague(DirichletCollection, (3, 3)), "s": vague(Categorical, 3)}
    args = hmm_arguments(model, init)
    assert np.allclose(args["A_prior"], 1.0) and np.allclose(args["B_init"], 1.0) and "A_known" not in args
    args = hmm_arguments(hidden_markov_model(p0=np.full(3, 1 / 3), A=PointMass(np.eye(3)), B=DirichletCollection(np.ones((4, 3)))),
                         {"B": vague(DirichletCollection, (4, 3))})
    assert np.allclose(args["A_known"], np.eye(3)) and args["B_prior"].shape == (4, 3)
    with pytest.raises(ValueError, match="initialization"):
        hmm_arguments(model, {"A": vague(DirichletCollection, (3, 3))})
    with pytest.raises(ValueError, match="shape"):
        hmm_arguments(model, {"A": vague(DirichletCollection, (3, 3)), "B": vague(DirichletCollection, (2, 3))})
    with pytest.raises(TypeError, match="DirichletCollection or PointMass"):
        hmm_arguments(hidden_markov_model(p0=np.full(3, 1 / 3), A=np.eye(3), B=PointMass(np.eye(3))), {})
    # infer refuses other factorisations and soft observations before it needs a device (context=object() would fail on
    # any use), so these run with and without a GPU
    from rxinfer_jl_b200 import MeanField
    for c in (MeanField(), None, "q(s)q(A)q(B)"):
        with pytest.raises(ValueError, match=r"q\(s, s_0\) q\(A\) q\(B\)"):
            rx.infer(model=model, data={"x": oh}, constraints=c, initialization=init, iterations=2, context=object())
    with pytest.raises(ValueError, match="one-hot"):
        rx.infer(model=model, data={"x": soft}, constraints=HMMConstraints(), initialization=init, iterations=2,
                 context=object())
    if not torch.cuda.is_available():
        # and needs a device otherwise (no CPU fallback)
        with pytest.raises(Exception):
            rx.infer(model=model, data={"x": oh}, constraints=HMMConstraints(), initialization=init, iterations=2)
