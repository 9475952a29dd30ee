"""rxg_hmm_vmp_f32 on the GPU: every chain gated against the fp64 reference of test_hmm.py, which gets the fp32-rounded
inputs.  Per chain: the Dirichlet parameters of q(A), q(B) (last iteration and KeepEach histories) at TOL_MEAN relative L2,
q(s_t), q(s_0) at 10 TOL_COV absolute, the free energy at FE_TOL relative to max(|F|, 1) per iteration and non-increasing.
Then long, sparse, near-deterministic and zero-containing inputs, flagged chains beside healthy ones, the reference test's
assertions on the CUDA output through infer, and the KeepEach histories against the last-iteration outputs bit for bit."""
import numpy as np
import pytest
import torch

from test_hmm import (MISSING, count_identities, gate, random_problem, reference_assertions, reference_data, reference_model,
                      reference_on_f32)
from util import TOL_COV, TOL_MEAN

pytestmark = pytest.mark.gpu
NB = 7                                         # odd batch
FE_TOL = 1e-5
LEARN = ((True, True), (True, False), (False, True), (False, False))


def run(ctx, x, kw, its, **extra):
    r = ctx.hmm_vmp(torch.as_tensor(x, device="cuda:0").contiguous(), **{k: np.asarray(v, np.float32) for k, v in kw.items()},
                    iterations=its, keep_each=True, **extra)
    return {k: (v.cpu().numpy() if v is not None else None) for k, v in r.items()}


def check(case, r, x, kw, its, chains=None):
    gate(case, r, reference_on_f32(x, kw, its), chains=chains, tol_mean=TOL_MEAN, tol_s=10 * TOL_COV, fe_tol=FE_TOL)


@pytest.mark.parametrize("K", [2, 3, 4, 5, 6, 7, 8])
def test_every_chain_against_the_fp64_reference(ctx, K):
    for M in (2, 5, 16):
        for T in (1, 7, 1000):
            for la, lb in LEARN:
                x, kw = random_problem(K, M, T, NB, seed=1000 * K + 10 * M + T + 2 * la + lb, learn_A=la, learn_B=lb,
                                       p_missing=0.1)
                for its in (1, 20):
                    check(f"K={K} M={M} T={T} its={its} learn A={la} B={lb}", run(ctx, x, kw, its), x, kw, its)


def test_cuda_output_keeps_the_column_convention(ctx):
    """Column sums of the A counts are the occupancies of s_0 .. s_{T-1}, row sums those of s_1 .. s_T; row sums of the B
    counts are the symbol counts (test_hmm.py::count_identities)."""
    count_identities(lambda x, kw, its: run(ctx, x, kw, its))


def test_long_chains_keep_log_z_accurate(ctx):
    """T = 10 000: log Z~ is a sum of 10^4 log c_t in fp64; the free energy stays at FE_TOL."""
    for la, lb in ((True, True), (False, False)):
        x, kw = random_problem(4, 5, 10000, 3, seed=11, learn_A=la, learn_B=lb)
        check(f"T=10000 learn A={la} B={lb}", run(ctx, x, kw, 5), x, kw, 5)


def test_sparse_sharp_and_zero_containing_inputs(ctx):
    # random missing steps, half of them
    x, kw = random_problem(5, 6, 300, NB, seed=12, p_missing=0.5)
    check("half missing", run(ctx, x, kw, 10), x, kw, 10)
    # a near-deterministic transition matrix (0.999 on the diagonal), known and learned
    for la in (False, True):
        x, kw = random_problem(3, 4, 500, NB, seed=13, learn_A=la, sharp=True)
        if la:
            kw["A_prior"] = kw["A_prior"] + 50.0 * np.eye(3)
        else:
            kw["A_known"] = 0.999 * np.eye(3) + 0.001 * np.roll(np.eye(3), 1, axis=0)
        check(f"sharp A learned={la}", run(ctx, x, kw, 8), x, kw, 8)
    # a known A with exact zeros (the reference's generating matrix), B learned, on the reference's data
    xr, _ = reference_data()
    A = np.array([[0.9, 0.0, 0.1], [0.1, 0.9, 0.0], [0.0, 0.1, 0.9]])
    kw = dict(p0=np.array([1.0, 0.0, 0.0]), A_known=A, B_prior=reference_model()["B_prior"], B_init=np.ones((3, 3)))
    x = np.repeat(xr[:, None], NB, 1)
    check("known A with zeros", run(ctx, x, kw, 6), x, kw, 6)


def test_flagged_chains_leave_their_neighbours_alone(ctx):
    x, kw = random_problem(3, 4, 50, NB, seed=14)
    x[10, 2] = 9                                               # a symbol >= M: RXG_ERR_BAD_ARG, read as missing
    r = run(ctx, x, kw, 4)
    assert list(r["status"]) == [0, 0, 1, 0, 0, 0, 0]
    xm = x.copy(); xm[10, 2] = MISSING
    check("bad symbol neighbours", r, xm, kw, 4, chains=[0, 1, 3, 4, 5, 6])
    # data impossible under known matrices: a zero normaliser flags RXG_ERR_NAN
    K = 3
    kwk = dict(p0=np.array([1.0, 0.0, 0.0]), A_known=np.roll(np.eye(K), 1, axis=0), B_known=np.eye(K))
    xi = np.tile(np.array([1, 2, 0, 1], np.uint8)[:, None], (1, NB))
    xi[:, 3] = [1, 2, 1, 0]
    r = run(ctx, xi, kwk, 1)
    assert list(r["status"]) == [0, 0, 0, 5, 0, 0, 0]
    check("impossible data neighbours", r, xi, kwk, 1, chains=[0, 1, 2, 4, 5, 6])


def test_reference_assertions_on_the_cuda_output_through_infer(ctx, rx):
    """hmm_tests.jl:36-96 with the reference's one-hot data, constraints, initialisation and returnvars."""
    from rxinfer_jl_b200 import Categorical, DirichletCollection, HMMConstraints, KeepEach, hidden_markov_model, vague
    xr, _ = reference_data()
    oh = torch.zeros(100, 3, NB)
    oh[torch.arange(100), torch.as_tensor(xr, dtype=torch.long), :] = 1.0
    ref = reference_model()
    model = hidden_markov_model(p0=ref["p0"], A=DirichletCollection(ref["A_prior"]), B=DirichletCollection(ref["B_prior"]))
    init = {"A": vague(DirichletCollection, (3, 3)), "B": vague(DirichletCollection, (3, 3)), "s": vague(Categorical, 3)}
    res = rx.infer(model=model, constraints=HMMConstraints(), data={"x": oh}, options={"limit_stack_depth": 500},
                   free_energy=True, initialization=init, iterations=20,
                   returnvars={"s": KeepEach(), "A": KeepEach(), "B": KeepEach()}, context=ctx)
    s, A, B = res.posteriors["s"].p, res.posteriors["A"].alpha, res.posteriors["B"].alpha
    fe = res.free_energy.cpu().numpy()
    assert s.shape == (20, 100, 3, NB) and A.shape == (20, 3, 3, NB) and B.shape == (20, 3, 3, NB)
    for b in range(NB):
        reference_assertions(s[..., b].cpu().numpy(), A[..., b], B[..., b], fe[:, b])
    assert res.posteriors["s_0"].p.shape == (3, NB)
    # the same data as uint8 symbols, KeepLast
    res2 = rx.infer(model=model, constraints=HMMConstraints(), data={"x": torch.as_tensor(np.repeat(xr[:, None], NB, 1))},
                    initialization=init, iterations=20, free_energy=True, context=ctx)
    assert torch.equal(res2.posteriors["s"].p, s[-1]) and torch.equal(res2.free_energy, res.free_energy)
    # flagged chains raise, as the other VMP models do
    bad = torch.as_tensor(np.repeat(xr[:, None], NB, 1)).clone()
    bad[4, 1] = 7
    with pytest.raises(rx.RxGaussError, match="1 of 7 chains"):
        rx.infer(model=model, constraints=HMMConstraints(), data={"x": bad}, initialization=init, iterations=2, context=ctx)


def test_keep_each_final_slot_equals_the_last_iteration_bit_for_bit(ctx):
    x, kw = random_problem(6, 9, 120, NB, seed=15, p_missing=0.2)
    xd = torch.as_tensor(x, device="cuda:0")
    k32 = {k: np.asarray(v, np.float32) for k, v in kw.items()}
    r = ctx.hmm_vmp(xd, **k32, iterations=7, keep_each=True)
    assert torch.equal(r["hist_s"][-1], r["s_prob"])
    assert torch.equal(r["hist_A"][-1], r["A_alpha"]) and torch.equal(r["hist_B"][-1], r["B_alpha"])
    r1 = ctx.hmm_vmp(xd, **k32, iterations=7, want_free_energy=False)
    assert r1["free_energy"] is None and "hist_s" not in r1
    assert torch.equal(r1["s_prob"], r["s_prob"]) and torch.equal(r1["A_alpha"], r["A_alpha"])


def test_c_entry_refusals(ctx, rx):
    x, kw = random_problem(3, 4, 10, 2, seed=16)
    xd = torch.as_tensor(x, device="cuda:0")
    k32 = {k: np.asarray(v, np.float32) for k, v in kw.items()}
    bad_cases = [dict(k32, A_known=np.eye(3, dtype=np.float32)),                         # both A choices
                 {k: v for k, v in k32.items() if k != "A_init"},                         # prior without init
                 dict(k32, A_prior=-k32["A_prior"]),                                      # Dirichlet parameter <= 0
                 dict(k32, p0=np.array([0.5, 0.5, 0.5], np.float32)),                     # p0 sums to 1.5
                 dict({k: v for k, v in k32.items() if not k.startswith("B")},
                      B_known=np.full((4, 3), 0.3, np.float32))]                          # columns sum to 1.2
    for c in bad_cases:
        with pytest.raises(rx.RxGaussError) as e:
            ctx.hmm_vmp(xd, **c)
        assert e.value.code == rx._lib.RXG_ERR_BAD_ARG, c
    x9, kw9 = random_problem(9, 3, 5, 2, seed=17)
    with pytest.raises(rx.RxGaussError) as e:
        ctx.hmm_vmp(torch.as_tensor(x9, device="cuda:0"), **kw9)
    assert e.value.code == rx._lib.RXG_ERR_UNSUPPORTED
    x17, kw17 = random_problem(2, 17, 5, 2, seed=18)
    with pytest.raises(rx.RxGaussError) as e:
        ctx.hmm_vmp(torch.as_tensor(x17, device="cuda:0"), **kw17)
    assert e.value.code == rx._lib.RXG_ERR_UNSUPPORTED
    with pytest.raises(ValueError, match="uint8"):
        ctx.hmm_vmp(xd.float(), **k32)
