"""wgmma descriptor / fragment plumbing self-test: D[128, n] = A[128, k] B[n, k]' on the tensor pipe with the 3xTF32 split must
match the fp64 product to fp32-level accuracy, for every operand shape the large-state sweeps issue
(K-major canonical layout with K = 16 / 32 / 64 / 128, N = 16 ... 128)."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

SHAPES = [(64, 128), (128, 64), (64, 64), (64, 32), (32, 32), (32, 16), (16, 16)]


@pytest.mark.parametrize("n,k", SHAPES)
def test_umma_tf32x3_matches_fp64(ctx, n, k):
    rng = np.random.default_rng(n * 1000 + k)
    A = rng.standard_normal((128, k)).astype(np.float32)
    B = rng.standard_normal((n, k)).astype(np.float32)
    D = ctx.selftest_umma(torch.as_tensor(A, device="cuda"), torch.as_tensor(B, device="cuda")).cpu().numpy()
    ref = A.astype(np.float64) @ B.astype(np.float64).T
    err = np.abs(D - ref).max() / np.abs(ref).max()
    assert err < 2e-6, err
    # structured probe: each output depends on one (row, col) pair only -> exact, catches any layout mix-up
    A2 = np.zeros((128, k), np.float32); B2 = np.zeros((n, k), np.float32)
    A2[np.arange(128), np.arange(128) % k] = np.arange(1, 129)
    B2[np.arange(n), (np.arange(n) * 3) % k] = 1.0 + np.arange(n)
    D2 = ctx.selftest_umma(torch.as_tensor(A2, device="cuda"), torch.as_tensor(B2, device="cuda")).cpu().numpy()
    assert np.array_equal(D2, A2.astype(np.float64) @ B2.astype(np.float64).T)


def test_umma_rejects_other_shapes(rx, ctx):
    with pytest.raises(rx.RxGaussError):
        ctx.selftest_umma(torch.zeros(128, 24, device="cuda"), torch.zeros(48, 24, device="cuda"))
