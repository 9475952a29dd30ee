"""The cluster sweep's per-chain covariances (`store_cov_span`, csrc/rxg_lgssm_cluster.cuh): each CTA writes one
contiguous span of the flattened cov[T][d][d][batch], not its own chains' pieces.

cov is filled with NaN inside guard regions of a sentinel value, through a 16-byte aligned view; after the sweep every
element must equal the de-duplicated `cov_shared_out=True` table bit for bit and the guards must be intact.  The batches
and T put span starts in the middle of rows and let one span cover many short rows (32 chains: a span is 32 rows of 8
float4s at T = 1) or at most two long ones (65 536 chains)."""
import pytest
import torch

from test_cluster_sweep_gpu import _lockstep, _smooth, max_T
from test_shared_sweep_variants import random_model

pytestmark = pytest.mark.gpu

GUARD = 64                  # floats on each side of the view (a multiple of 4: the view stays 16-byte aligned)
SENTINEL = -12345.0


@pytest.mark.parametrize("batch", [32, 96, 160, 65536])
@pytest.mark.parametrize("d", [1, 2, 3, 4])
def test_spans_equal_the_shared_table(ctx, d, batch):
    mod = random_model(d, d, seed=9000 + d)
    g = torch.Generator(device="cuda").manual_seed(d * batch)
    for T in (1, 17, 129, 1000, max_T(d, d)):
        case = f"d={d} batch={batch} T={T}"
        y = torch.randn(T, d, batch, device="cuda", generator=g) * 3.0
        ls, launches_ls = _lockstep(ctx, y, mod)
        del ls
        n = T * d * d * batch
        buf = torch.full((n + 2 * GUARD,), float("nan"), device="cuda")
        buf[:GUARD] = SENTINEL
        buf[-GUARD:] = SENTINEL
        cov = buf[GUARD:GUARD + n].view(T, d, d, batch)
        assert cov.data_ptr() % 16 == 0
        r, launches = _smooth(ctx, y, mod, out_cov=cov)
        assert launches == launches_ls + 1, f"{case}: the cluster sweep did not run"
        tab, _ = _smooth(ctx, y, mod, cov_shared_out=True)
        assert torch.equal(cov, tab["cov"][..., None].expand(T, d, d, batch)), f"{case}: covariances differ from the table"
        assert bool((buf[:GUARD] == SENTINEL).all()) and bool((buf[-GUARD:] == SENTINEL).all()), f"{case}: guard overwritten"
        assert torch.equal(r["mean"], tab["mean"]), f"{case}: means differ between the two outputs"
        del y, buf, cov, r, tab
