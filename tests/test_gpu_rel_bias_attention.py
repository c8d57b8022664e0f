"""The research-path relative-bias attention (the generic kernels of csrc/attn_generic.cu with pos_w / ts_w) against the fp64
oracle, at the shapes of the benchmarked research configurations and across tiles, in fp32, bf16 and fp16; and the research
block itself in bf16 at the two benchmarked configurations.

The bias-table gradients are the delicate part of the dQ kernel: per tile pair, the position-bias gradient of its 2 TILE - 1
diagonals is gathered in shared memory and flushed to pos_w entry n - 1 + (n0 - m0) + t - (TILE - 1); the time-bias gradient
goes through a per-CTA histogram after a warp pre-sum when all lanes share a bucket.  They are judged entry by entry against
the oracle (bound: tests/util.py table_bound), band by band of 64 diagonals, and the j > i diagonals must stay exactly zero.
Inputs are rounded to the kernel's dtype first and the oracle runs in fp64 on those values, so only the kernel's own
arithmetic and the storage rounding of its outputs are measured.
"""
import pytest
import torch

from util import (TOL, assert_pos_bands, assert_rel, assert_rel_segments, assert_table_entries, assert_zero_from,
                  offsets_from, rel_bias_reference, research_case, research_reference, table_bound)

pytestmark = pytest.mark.gpu
DEV = "cuda"
H = 3
DIMS = [(8, 8), (32, 32), (24, 40), (96, 96), (160, 160)]  # amzn_books, ml20m, dqk != dv, DMAX 128, DMAX 256 (TILE 32 backward)


def _lengths(n):
    """Sequence lengths of one batch: empty, single row, both sides of the 64-row tile edge, n - 1 and n."""
    return [x for x in (65, 0, n, 1, 63, n - 1, 64) if x <= n]


def _timestamps(kind, B, n, g):
    if kind == "bench":  # cumulative gaps of up to one day, as in the benchmark's data
        return torch.randint(0, 86400, (B, n), generator=g).cumsum(1), 128
    # non-monotone, with repeats (bucket 0) and jumps up to 1e9 s: most pairs clamp to the last of 16 buckets
    ts = torch.randint(0, 3, (B, n), generator=g).cumsum(1)
    jump = torch.rand(B, n, generator=g) < 0.15
    ts = ts + jump * torch.randint(-10**9, 10**9, (B, n), generator=g)
    return ts, 16


def _case(dtype, dqk, dv, n, bias, seed):
    g = torch.Generator().manual_seed(seed)
    lengths = _lengths(n)
    off = offsets_from(lengths)
    L = int(off[-1])
    s = dqk ** -0.25  # q.k has an rms of 1 (alpha = 1 on the research path)
    q, k = ((s * torch.randn(L, H, dqk, generator=g)).to(dtype) for _ in range(2))
    v, dout = (torch.randn(L, H, dv, generator=g).to(dtype) for _ in range(2))
    pos_w = (0.5 * torch.randn(2 * n - 1, generator=g)).to(dtype)
    ts_w = ts = None
    if bias != "pos":
        ts, nb = _timestamps(bias, len(lengths), n, g)
        ts_w = (0.5 * torch.randn(nb + 1, generator=g)).to(dtype)
    return q, k, v, dout, off, pos_w, ts_w, ts


def _kernel(n, q, k, v, dout, off, pos_w, ts_w, ts):
    from generative_recommenders_b200 import _lib
    from generative_recommenders_b200.ops.hstu_attention import cuda_hstu_attention_bwd, cuda_hstu_attention_fwd

    qd, kd, vd, dod, offd = (t.to(DEV) for t in (q, k, v, dout, off))
    bias = (pos_w.to(DEV), None if ts_w is None else ts_w.to(DEV), None if ts is None else ts.to(DEV))
    out = cuda_hstu_attention_fwd(n, 1.0, qd, kd, vd, offd, impl=_lib.IMPL_GENERIC, bias=bias)
    dq, dk, dv = torch.empty_like(qd), torch.empty_like(kd), torch.empty_like(vd)
    dpos = torch.zeros(2 * n - 1, dtype=torch.float32, device=DEV)
    dts = None if ts_w is None else torch.zeros(ts_w.numel(), dtype=torch.float32, device=DEV)
    cuda_hstu_attention_bwd(n, 1.0, dod, qd, kd, vd, dq, dk, dv, offd, impl=_lib.IMPL_GENERIC, bias=bias, dbias=(dpos, dts),
                            deterministic=False)
    return out, dq, dk, dv, dpos, dts


@pytest.mark.parametrize("bias", ["pos", "bench", "adversarial"])
@pytest.mark.parametrize("n", [61, 129, 211])
@pytest.mark.parametrize("dqk,dv", DIMS)
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16], ids=["fp32", "bf16", "fp16"])
def test_rel_bias_attention_fwd_bwd(dtype, dqk, dv, n, bias):
    q, k, v, dout, off, pos_w, ts_w, ts = _case(dtype, dqk, dv, n, bias, seed=n * 1000 + dqk + dv)
    out, dq, dk, dv_, dpos, dts = _kernel(n, q, k, v, dout, off, pos_w, ts_w, ts)
    ref = rel_bias_reference(n, q, k, v, dout, off, pos_w, ts_w, ts)
    for name, got in (("out", out), ("dq", dq), ("dk", dk), ("dv", dv_)):
        assert_rel_segments(got, ref[name], off, n, f"{name}")
    assert_zero_from(dpos, n, "dpos_w (j > i diagonals)")
    d = max(dqk, dv)
    assert_table_entries(dpos, ref["dpos"], table_bound(ref["mass_pos"], ref["cnt_pos"], d), "dpos_w")
    # dpos_w is accumulated in fp32: the fp32 bound on every band of 64 diagonals
    assert_pos_bands(dpos, ref["dpos"], n, TOL[torch.float32], "dpos_w")
    if ts_w is not None:
        assert_table_entries(dts, ref["dts"], table_bound(ref["mass_ts"], ref["cnt_ts"], d), "dts_w")
        if bias == "adversarial":
            assert ref["cnt_ts"][-1] > 0 and ref["cnt_ts"][0] > 0, "the case must reach bucket 0 and the clamped last bucket"


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16], ids=["fp32", "bf16", "fp16"])
def test_rel_bias_attention_autograd_returns_tables_in_parameter_dtype(dtype):
    from generative_recommenders_b200.ops.hstu_attention import hstu_rel_bias_attention

    n = 129
    q, k, v, dout, off, pos_w, ts_w, ts = _case(dtype, 32, 32, n, "bench", seed=7)
    leaves = [t.to(DEV).requires_grad_() for t in (q, k, v, pos_w, ts_w)]
    out = hstu_rel_bias_attention(n, *leaves[:3], off.to(DEV), leaves[3], leaves[4], ts.to(DEV))
    out.backward(dout.to(DEV))
    ref = rel_bias_reference(n, q, k, v, dout, off, pos_w, ts_w, ts)
    for leaf, name in zip(leaves, ("dq", "dk", "dv", "dpos", "dts")):
        assert leaf.grad is not None and leaf.grad.dtype == dtype, (name, None if leaf.grad is None else leaf.grad.dtype)
    for leaf, name in zip(leaves[:3], ("dq", "dk", "dv")):
        assert_rel(leaf.grad, ref[name], name)
    # the tables are accumulated in fp32 and cast to the parameter dtype: the fp32 bound plus that storage rounding
    assert_rel(leaves[3].grad, ref["dpos"], "dpos_w", tol=TOL[torch.float32])
    assert_rel(leaves[4].grad, ref["dts"], "dts_w", tol=TOL[torch.float32])
    assert_zero_from(leaves[3].grad, n, "dpos_w (j > i diagonals)")


# ------------------------------------------------------------------------------------------------------------------
# the research block in bf16 at the benchmarked configurations (B reduced so that the fp64 oracle stays fast)
# ------------------------------------------------------------------------------------------------------------------
def _block(c):
    from generative_recommenders_b200.modules.research_hstu import (
        RelativeBucketedTimeAndPositionBasedBias,
        SequentialTransductionUnitJagged,
    )

    blk = SequentialTransductionUnitJagged(
        embedding_dim=c["D"], linear_hidden_dim=c["dv"], attention_dim=c["dqk"], dropout_ratio=0.0, attn_dropout_ratio=0.0,
        num_heads=c["H"], linear_activation="silu",
        relative_attention_bias_module=RelativeBucketedTimeAndPositionBasedBias(max_seq_len=c["n"], num_buckets=128),
        normalization="rel_bias", linear_config="uvqk", concat_ua=c["concat_ua"], epsilon=1e-6, max_length=c["n"],
    ).to(torch.bfloat16)
    blk.load_state_dict(c["params"], strict=True)
    return blk.to(DEV)


@pytest.mark.parametrize("concat_ua", [False, True], ids=["plain", "concat_ua"])
@pytest.mark.parametrize("config", ["ml20m", "amzn_books"])
def test_research_block_bf16_at_bench_shapes(config, concat_ua):
    c = research_case(config, concat_ua)
    blk = _block(c)
    x = c["x"].to(DEV).requires_grad_()
    n = c["n"]
    y, _ = blk(x, c["seq_offsets"].to(DEV), c["timestamps"].to(DEV), torch.tril(torch.ones(n, n, device=DEV)))
    y.backward(c["dy"].to(DEV))
    staged, exact, dist = research_reference(c)
    # forward: the oracle with bf16 rounding at the boundaries the module stores, so the north-star bound applies unchanged
    assert_rel(y, staged["y"], f"{config} y")
    # gradients against fp64: at most twice the staged oracle's own distance from fp64 (measured on these inputs, and pinned
    # in test_research_checkers_cpu.py), never less than the fp32 bound (the o.bias gradient does not depend on the forward:
    # its distance is 0), plus the storage rounding of the gradient itself
    grads = dict(x=x.grad, **{k: p.grad for k, p in blk.named_parameters()})
    for name, ref in exact.items():
        if name == "y":
            continue
        got = grads[name]
        assert got is not None and got.dtype == torch.bfloat16, name
        assert_rel(got, ref, f"{config} d{name}", tol=max(2 * dist[name], TOL[torch.float32]))
