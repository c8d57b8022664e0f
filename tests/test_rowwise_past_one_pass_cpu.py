"""The checks of test_gpu_rowwise_past_one_pass.py have teeth (CPU, oracle only).  The "kernel outputs" are the fp64 oracle
rounded to bf16, and each test feeds a check a copy that is wrong the way a persistent kernel could be wrong past its first
grid pass:

- the explicit fp64 oracle of the output stage agrees with torch autograd through hstu_oracle's forward, dropout included;
- a block that uses the neighbouring row's rstd passes the whole-tensor bound and fails the per-block one, which names it;
- dw / db summed only from the last row each backward warp handles, as a per-row reset of the kernel's register
  accumulators would leave them, fail the fp32 bound;
- the mask statistics accept an i.i.d. Bernoulli mask and reject one whose second pass (of the backward or of the forward
  grid) repeats its first.
"""
import pytest
import torch

import test_gpu_rowwise_past_one_pass as P
from oracle import hstu_oracle as O
from util import BLOCK_ROWS, TOL, assert_rel, assert_rel_blocks

BF16 = torch.bfloat16


@pytest.mark.parametrize("silu_u", [False, True])
@pytest.mark.parametrize("concat", [0, 1, 2])
def test_explicit_oracle_matches_autograd(concat, silu_u):
    n, p = 300, 0.3
    attn, u, w, b, dout = P._inputs(n, concat, BF16, seed=5 + concat)
    keep = torch.rand(dout.shape, generator=torch.Generator().manual_seed(6)) >= p
    out, dattn, du, dw, db, mean, rstd = P.nmd_oracle(attn, u, w, b, dout, keep, p, silu_u, concat)
    a64, u64, w64, b64 = (t.double().requires_grad_() for t in (attn, u, w, b))
    if concat < 2:
        ref = O.norm_mul_dropout_fwd(a64, u64, w64, b64, P.EPS, silu_u=silu_u, concat_ux=concat == 1, dtype=torch.float64)
    else:  # concat_ua of the research block: the middle part is LN(attn)
        uf = torch.nn.functional.silu(u64) if silu_u else u64
        nrm = O.layer_norm_fwd(a64, w64, b64, P.EPS, dtype=torch.float64)[0]
        ref = torch.cat([uf, nrm, uf * nrm], 1)
    ref = ref * keep.double() / (1 - p)
    ref.backward(dout.double())
    _, mr, rr = O.layer_norm_fwd(attn, None, None, P.EPS, dtype=torch.float64)
    for name, got, r in (("out", out, ref.detach()), ("dattn", dattn, a64.grad), ("du", du, u64.grad), ("dw", dw, w64.grad),
                         ("db", db, b64.grad), ("mean", mean, mr), ("rstd", rstd, rr)):
        assert torch.allclose(got, r, rtol=1e-12, atol=1e-12), name


def _spread_rows(n, seed):
    """attn whose rows have exact standard deviations exp(0.002 N(0, 1)): neighbouring rows' rstd differ by about 0.3 %."""
    g = torch.Generator().manual_seed(seed)
    z = torch.randn(n, P.W, generator=g, dtype=torch.float64)
    z = (z - z.mean(1, keepdim=True)) / z.std(1, unbiased=False, keepdim=True)
    s = torch.exp(0.002 * torch.randn(n, 1, generator=g, dtype=torch.float64))
    return (z * s + 0.1 * torch.randn(n, 1, generator=g, dtype=torch.float64)).to(BF16)


def test_neighbour_rstd_in_one_block_passes_globally_and_fails_its_block():
    n = P.N_BENCH
    attn = _spread_rows(n, 11)
    _, u, w, b, dout = P._inputs(n, 0, BF16, seed=12)
    ref, _, _, _, _, mean, rstd = P.nmd_oracle(attn, u, w, b, dout, None, 0.0, False, 0)
    assert_rel_blocks(ref.to(BF16), ref, "rounded oracle")
    r0, r1 = 5 * BLOCK_ROWS, 6 * BLOCK_ROWS
    a, uu, w64, b64 = (t.double() for t in (attn[r0:r1], u[r0:r1], w, b))
    nb = rstd[r0 + 1:r1 + 1].unsqueeze(1)  # the next row's rstd
    bad = ref.clone()
    bad[r0:r1] = uu * ((a - mean[r0:r1].unsqueeze(1)) * nb * w64 + b64)
    bad = bad.to(BF16)
    assert_rel(bad, ref, "neighbour rstd in one block, whole tensor")
    with pytest.raises(AssertionError, match=rf"rows \[{r0}, {r1}\)"):
        assert_rel_blocks(bad, ref, "neighbour rstd in one block")


def test_dw_db_from_each_warps_last_row_only_fail():
    """The backward's row -> (CTA, warp) map: r = (step x 528 + cta) x 8 + warp, so the warp slot of row r is r mod 4,224 and
    its last row is the largest such r below n."""
    n, p, concat = P.N_GRID, 0.2, 1
    attn, u, w, b, dout = P._inputs(n, concat, BF16, seed=21)
    keep = torch.rand(dout.shape, generator=torch.Generator().manual_seed(22)) >= p
    last = torch.arange(n) >= n - BLOCK_ROWS  # rows with no row of the same warp slot after them
    dw = db = dw_last = db_last = 0.0
    for r0 in range(0, n, P.CHUNK):
        r1 = min(n, r0 + P.CHUNK)
        *_, dwc, dbc, _, _ = P.nmd_oracle(attn[r0:r1], u[r0:r1], w, b, dout[r0:r1], keep[r0:r1], p, False, concat)
        lr = last[r0:r1]
        dw, db = dw + dwc, db + dbc
        if lr.any():
            *_, dwl, dbl, _, _ = P.nmd_oracle(attn[r0:r1][lr], u[r0:r1][lr], w, b, dout[r0:r1][lr], keep[r0:r1][lr], p, False,
                                              concat)
            dw_last, db_last = dw_last + dwl, db_last + dbl
    f32 = TOL[torch.float32]
    assert_rel(dw.float(), dw, "dw of all rows", tol=f32)
    assert_rel(db.float(), db, "db of all rows", tol=f32)
    for name, got, ref in (("dw", dw_last, dw), ("db", db_last, db)):
        with pytest.raises(AssertionError, match="rel-L2 error"):
            assert_rel(got.float(), ref, f"{name} of each warp's last row", tol=f32)


def _bernoulli(n, K, p, seed):
    return torch.rand(n, K, generator=torch.Generator().manual_seed(seed)) >= p


@pytest.mark.parametrize("K", [P.W, 3 * P.W])
def test_mask_statistics_accept_iid_bernoulli(K):
    P.check_mask_stats(_bernoulli(P.N_BENCH, K, 0.2, K), 0.2, "i.i.d. Bernoulli")


@pytest.mark.parametrize("K", [P.W, 3 * P.W])
@pytest.mark.parametrize("shift", [P.BWD_PASS, P.FWD_PASS])
def test_mask_statistics_reject_a_repeated_second_pass(shift, K):
    keep = _bernoulli(P.N_BENCH, K, 0.2, 3 + K)
    keep[shift:2 * shift] = keep[:shift]
    with pytest.raises(AssertionError, match=f"rows r and r \\+ {shift} agree"):
        P.check_mask_stats(keep, 0.2, "second pass repeats the first")
