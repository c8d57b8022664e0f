"""Attention on the wgmma kernels when the value head is wider than the query / key head (dqk < dv), bf16 and fp16.

AUTO runs attn_fwd_mixed_wgmma_kernel, attn_fwd_delta_mixed_wgmma_kernel (with delta_reduce_kernel when the keys are split
into chunks) and, for the backward, attn_bwd_dkdv_mixed_wgmma_kernel + attn_bwd_dq_mixed_wgmma_kernel.  Checked against the
fp64 oracle on the whole tensor (assert_rel) and per 64-row segment (assert_rel_segments): every pair, the mask options,
lengths around the tiles with rows past max_seq_len, the score-scale sweep at (128, 256), strided views of one buffer,
delta-q with and without key chunks, the KV-cached STULayer, a bf16 STUStack at attention_dim 128 / hidden_dim 256, and
bitwise repeatability of the backward (no atomics).
"""
import ctypes as C

import pytest
import torch

from oracle import hstu_oracle as O
from test_gpu_attention import _random_case
from test_gpu_attention_deterministic import _kernels_of
from test_gpu_attention_numerics import SIGMAS, _compare, _oracle, _run
from util import assert_rel, assert_rel_segments, offsets_from

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda")
PAIRS = [(32, 64), (32, 128), (32, 256), (64, 128), (64, 256), (128, 256)]
DTYPES = [torch.bfloat16, torch.float16]
FWD = "attn_fwd_mixed_wgmma_kernel"
BWD = ("attn_bwd_dkdv_mixed_wgmma_kernel", "attn_bwd_dq_mixed_wgmma_kernel")
GENERIC = "generic"


def _lib():
    from generative_recommenders_b200 import _lib

    return _lib


def _case(lengths, targets, H, dqk, dv, sigma, dtype, seed, i32=False):
    """q, k ~ N(0, sigma^2) [L, H, dqk]; v, dout ~ N(0, 1) [L, H, dv]; with alpha = 1/sqrt(dqk), rms(alpha S) = sigma^2."""
    g = torch.Generator().manual_seed(seed)
    idt = torch.int32 if i32 else torch.int64
    off = offsets_from(lengths, dtype=idt)
    L = int(off[-1])
    q, k = ((sigma * torch.randn(L, H, dqk, generator=g)).to(dtype) for _ in range(2))
    v, dout = (torch.randn(L, H, dv, generator=g).to(dtype) for _ in range(2))
    return q, k, v, dout, off, None if targets is None else torch.tensor(targets, dtype=idt)


def _bwd(N, alpha, do, q, k, v, off, nt, win=0, ctx=0, min_full=0, grads=None):
    from generative_recommenders_b200.ops import hstu_attention as ha

    dq, dk, dv = grads if grads is not None else (torch.full_like(t, float("nan")) for t in (q, k, v))
    ha.cuda_hstu_attention_bwd(N, alpha, do, q, k, v, dq, dk, dv, off, num_targets=nt, max_attn_len=win,
                               contextual_seq_len=ctx, min_full_attn_seq_len=min_full, deterministic=False)
    return dq, dk, dv


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("dqk,dv", PAIRS)
def test_mixed_dims_select_and_run_the_wgmma_kernels(dqk, dv, dtype):
    from generative_recommenders_b200.ops import hstu_attention as ha

    _l = _lib()
    q, k, v, do, off, nt = (t.to(DEV) for t in _case([300, 129], [3, 1], 2, dqk, dv, 0.8, dtype, dqk + dv))
    N, alpha = 320, dqk**-0.5
    p = _l.AttnParams()
    ha._fill_common(p, N, alpha, q, k, v, off, None, 0, 0, 0, _l.IMPL_AUTO)
    out = torch.empty(q.shape[0], 2, dv, device=DEV, dtype=dtype)
    p.out, p.o_row_stride, p.o_head_stride = out.data_ptr(), out.stride(0), out.stride(1)
    lib = _l.lib()
    assert lib.hstu_attn_select_impl(C.byref(p), 0) == _l.IMPL_UMMA
    assert lib.hstu_attn_workspace_bytes(C.byref(p), 0) == 0
    p.dout, p.dq, p.dk, p.dv_out = do.data_ptr(), q.data_ptr(), k.data_ptr(), v.data_ptr()
    for name, t in (("do", do), ("dq", q), ("dk", k), ("dv", v)):
        setattr(p, f"{name}_row_stride", t.stride(0))
        setattr(p, f"{name}_head_stride", t.stride(1))
    assert lib.hstu_attn_select_impl(C.byref(p), 1) == _l.IMPL_UMMA
    assert lib.hstu_attn_workspace_bytes(C.byref(p), 1) == 0
    # both directions run and write finite results (which kernels run is shown by the STUStack test below)
    got = _run(_l.IMPL_AUTO, N, alpha, q, k, v, do, off, nt)
    torch.cuda.synchronize()
    for t in got:
        assert torch.isfinite(t).all()


MASK_OPTS = [(False, False, 0, 0, False), (True, False, 0, 0, False), (True, True, 5, 33, False), (False, False, 4, 0, False),
             (True, False, 0, 0, True), (True, True, 5, 33, True)]


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("dqk,dv", PAIRS)
@pytest.mark.parametrize("opts", MASK_OPTS)
def test_mixed_dims_mask_options_vs_oracle(dqk, dv, dtype, opts):
    """Plain causal, targets, a window with min_full_attn_seq_len, a contextual prefix and int32 offsets."""
    targets, window, ctx, min_full, i32 = opts
    c = _random_case(31 * dqk + dv + ctx, dtype, 4, 2, 260, 24, dqk, dv, targets, window, ctx, min_full, i32=i32)
    args = (c["max_seq_len"], c["alpha"], c["q"], c["k"], c["v"], c["dout"], c["seq_offsets"], c["num_targets"],
            c["max_attn_len"], c["contextual_seq_len"], c["min_full_attn_seq_len"])
    got = _run(_lib().IMPL_UMMA, *args)
    ref = _oracle(c["max_seq_len"], c["alpha"], c["q"], c["k"], c["v"], c["dout"], c["seq_offsets"].long(),
                  None if c["num_targets"] is None else c["num_targets"].long(), *args[8:])
    _compare(got, ref, c["seq_offsets"], c["max_seq_len"], f"({dqk}, {dv}) {dtype} {opts}")


@pytest.mark.parametrize("dtype,i32", [(torch.bfloat16, True), (torch.float16, False)])
@pytest.mark.parametrize("dqk,dv", PAIRS)
def test_mixed_dims_lengths_and_rows_past_max_seq_len(dqk, dv, dtype, i32):
    """Lengths 0, 1, 63, 64, 65, 127, 128, 129, one of max_seq_len and one past it, whose rows past max_seq_len must be exact
    zeros in out, dq, dk and dv: the allocator is filled with NaN first, and the gradient buffers start as NaN."""
    lengths, targets, N = [640, 0, 1, 63, 64, 65, 127, 128, 129, 700], [9, 0, 1, 3, 0, 5, 1, 2, 7, 4], 640
    alpha = dqk**-0.5
    q, k, v, do, off, nt = _case(lengths, targets, 2, dqk, dv, 0.8, dtype, 77 + dqk + dv, i32=i32)
    poison = torch.full((64 << 20,), float("nan"), device=DEV)
    del poison
    got = _run(_lib().IMPL_AUTO, N, alpha, q, k, v, do, off, nt)
    torch.cuda.synchronize()
    ref = _oracle(N, alpha, q, k, v, do, off.long(), nt.long())
    _compare(got, ref, off, N, f"lengths ({dqk}, {dv}) {dtype}")
    last = slice(int(off[-2]) + N, int(off[-1]))
    for name, a in zip(("out", "dq", "dk", "dv"), got):
        assert torch.equal(a[last].float().cpu(), torch.zeros_like(a[last].float().cpu())), f"{name}: rows past max_seq_len"


@pytest.mark.parametrize("sigma", SIGMAS)
@pytest.mark.parametrize("dtype", DTYPES)
def test_mixed_dims_across_score_scales(sigma, dtype):
    """(128, 256) at rms(alpha S) = 0.09, 1, 2.25 and 4: the per-segment error stays inside the bound at every scale."""
    dqk, dv, N = 128, 256, 1536
    q, k, v, do, off, nt = _case([1500, 731, 260, 1], [7, 3, 0, 1], 2, dqk, dv, sigma, dtype, 2024 + dqk)
    got = _run(_lib().IMPL_UMMA, N, dqk**-0.5, q, k, v, do, off, nt)
    ref = _oracle(N, dqk**-0.5, q, k, v, do, off, nt)
    _compare(got, ref, off, N, f"(128, 256) {dtype} rms(alpha S)={sigma**2:g}")


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("dqk,dv", [(32, 256), (64, 128), (128, 256)])
def test_mixed_dims_strided_views_of_one_buffer(dqk, dv, dtype):
    """q, k, v as strided views of one [L, H, 2 dqk + dv] buffer and dq, dk, dv of one NaN-filled gradient buffer, with
    targets, a window, a full-attention tail, a contextual prefix, int32 offsets, an empty sequence, a length-1 sequence
    and a sequence past max_seq_len."""
    lengths, targets, N, win, min_full, ctx = [700, 0, 1, 517, 300], [9, 0, 1, 4, 2], 640, 150, 64, 37
    H, alpha = 2, dqk**-0.5
    q, k, v, do, off, nt = _case(lengths, targets, H, dqk, dv, 1.0, dtype, 357, i32=True)
    L = q.shape[0]
    buf = torch.empty(L, H, 2 * dqk + dv, device=DEV, dtype=dtype)
    qd, kd, vd = torch.split(buf, [dqk, dqk, dv], dim=2)
    for dst, src in zip((qd, kd, vd), (q, k, v)):
        dst.copy_(src)
    gbuf = torch.full((L, H, 2 * dqk + dv), float("nan"), device=DEV, dtype=dtype)
    grads = torch.split(gbuf, [dqk, dqk, dv], dim=2)
    out = _run(_lib().IMPL_AUTO, N, alpha, qd, kd, vd, do, off, nt, win, ctx, min_full, bwd=False)[0]
    got = _bwd(N, alpha, do.to(DEV), qd, kd, vd, off.to(DEV), nt.to(DEV), win, ctx, min_full, grads=grads)
    torch.cuda.synchronize()
    ref = _oracle(N, alpha, q, k, v, do, off.long(), nt.long(), win, ctx, min_full)
    _compare((out,) + tuple(got), ref, off, N, f"strided ({dqk}, {dv}) {dtype}")


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("dqk,dv", PAIRS)
def test_mixed_dims_empty_batch(dqk, dv, dtype):
    """L == 0: nothing to compute, and nothing fails."""
    q, k, v, do, off, nt = _case([0, 0], None, 2, dqk, dv, 1.0, dtype, 1)
    got = _run(_lib().IMPL_AUTO, 64, dqk**-0.5, q, k, v, do, off, nt)
    assert all(t.shape[0] == 0 for t in got)


def _delta_case(B, n_cache, delta, H, dqk, dv, dtype, seed):
    lengths = [n_cache + delta - (7 * b) % 50 for b in range(B)]
    q, k, v, _, off, _ = _case(lengths, None, H, dqk, dv, 0.8, dtype, seed)
    rows = torch.cat([torch.arange(int(off[b + 1]) - delta, int(off[b + 1])) for b in range(B)])
    nt = torch.full((B,), delta, dtype=torch.int64)
    return q[rows], k, v, off, nt, max(lengths)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("dqk,dv", PAIRS)
@pytest.mark.parametrize("B,n_cache", [(1, 4000), (128, 300)])
def test_mixed_dims_delta_q_vs_oracle(dqk, dv, dtype, B, n_cache):
    """delta_hstu_mha against the oracle: B = 1 on a 4000-key cache splits the keys into chunks (fp32 partials and
    delta_reduce_kernel), B = 128 runs one chunk, whose kernel writes out itself."""
    from generative_recommenders_b200.ops.hstu_attention import delta_hstu_mha

    delta = 16
    dq_, k, v, off, nt, N = _delta_case(B, n_cache, delta, 2, dqk, dv, dtype, dqk * dv + B)
    alpha = dqk**-0.5
    res = {}
    names = _kernels_of(lambda: res.setdefault("out", delta_hstu_mha(N, alpha, dq_.to(DEV), k.to(DEV), v.to(DEV),
                                                                     off.to(DEV), num_targets=nt.to(DEV))))
    assert any("attn_fwd_delta_mixed_wgmma_kernel" in n for n in names), sorted(names)
    assert any("delta_reduce_kernel" in n for n in names) == (B == 1), sorted(names)
    ref = O.delta_hstu_mha_fwd(N, alpha, dq_, k, v, off, num_targets=nt, dtype=torch.float64)
    assert_rel(res["out"], ref, f"delta ({dqk}, {dv}) {dtype} B={B}")


def test_stu_layer_cached_forward_at_attention_128_hidden_256():
    """STULayer(attention_dim=128, hidden_dim=256), bf16: prefill, then cached_forward on the last rows, matches the full
    forward on those rows, with the delta-q forward on the wgmma kernels."""
    from generative_recommenders_b200.modules.stu import STULayer, STULayerConfig, STUStack

    torch.manual_seed(5)
    D, H, delta = 256, 2, 16
    stack = STUStack([STULayer(STULayerConfig(embedding_dim=D, num_heads=H, hidden_dim=256, attention_dim=128,
                                              output_dropout_ratio=0.0, target_aware=True))])
    stack = stack.to(DEV).to(torch.bfloat16).eval()
    lengths = torch.tensor([700, 129, 1000, 64], device=DEV)
    full_len = lengths + delta
    nt = torch.full((4,), delta, device=DEV)
    off = offsets_from(full_len.tolist(), DEV)
    N = 1000 + delta
    x = torch.randn(int(off[-1]), D, device=DEV).to(torch.bfloat16)
    with torch.no_grad():
        y_full = stack(x=x, x_lengths=full_len, x_offsets=off, max_seq_len=N, num_targets=nt)
        for layer in stack._stu_layers:
            layer.reset_kv_cache()
        stack(x=x, x_lengths=full_len, x_offsets=off, max_seq_len=N, num_targets=nt, max_kv_caching_len=1000,
              kv_caching_lengths=lengths)
        rows = torch.cat([torch.arange(int(off[i + 1]) - delta, int(off[i + 1]), device=DEV) for i in range(4)])
        res = {}
        names = _kernels_of(lambda: res.setdefault("y", stack.cached_forward(delta_x=x[rows], num_targets=nt)))
    assert any("attn_fwd_delta_mixed_wgmma_kernel" in n for n in names), sorted(names)
    assert not any("generic" in n for n in names), sorted(names)
    assert_rel(res["y"], y_full[rows].float(), "cached vs full forward, (128, 256) bf16", tol=1.5e-2)


def test_stu_stack_bf16_at_attention_128_hidden_256():
    """A bf16 STUStack with attention_dim = 128 and hidden_dim = 256: its attention runs on the wgmma kernels forward and
    backward, the forward matches the fp32 oracle within the bf16 stack budget (1.5e-2) and the gradients are finite."""
    from generative_recommenders_b200.modules.stu import STULayer, STULayerConfig, STUStack

    torch.manual_seed(23)
    Dm, H, N = 256, 2, 1024
    lengths, nts = [1024, 700, 129], [7, 2, 1]
    off = offsets_from(lengths)
    L = int(off[-1])
    stack = STUStack([STULayer(STULayerConfig(embedding_dim=Dm, num_heads=H, hidden_dim=256, attention_dim=128,
                                              output_dropout_ratio=0.0, target_aware=True)) for _ in range(2)])
    stack = stack.to(DEV).to(torch.bfloat16)
    x = torch.randn(L, Dm).to(torch.bfloat16)
    xd = x.to(DEV).requires_grad_()
    out = {}

    def run():
        y = stack(x=xd, x_lengths=torch.tensor(lengths, device=DEV), x_offsets=off.to(DEV), max_seq_len=N,
                  num_targets=torch.tensor(nts, device=DEV))
        y.float().square().mean().backward()
        out["y"] = y

    names = _kernels_of(run)
    for kname in (FWD,) + BWD:
        assert any(kname in n for n in names), (kname, sorted(names))
    assert not any("attn_fwd_generic" in n or "attn_bwd_kv_generic" in n for n in names), sorted(names)
    assert torch.isfinite(xd.grad).all()
    for n, p in stack.named_parameters():
        assert p.grad is not None and torch.isfinite(p.grad).all(), n
    sd = {k: v.detach().float().cpu() for k, v in stack.state_dict().items()}
    h = x.float()
    for layer in range(2):
        p = {k.split(".")[-1]: v for k, v in sd.items() if k.startswith(f"_stu_layers.{layer}.")}
        h = O.stu_layer_fwd(h, off, N, torch.tensor(nts), p, H, 128, 256)
    assert_rel(out["y"], h, "STUStack (128, 256) bf16 y", tol=1.5e-2)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("dqk,dv", PAIRS)
def test_mixed_dims_backward_is_bitwise_repeatable(dqk, dv, dtype):
    """No atomics in either kernel: two identical calls give bitwise-equal dq, dk and dv."""
    N = 2048
    q, k, v, do, off, nt = (t.to(DEV) for t in _case([N, N - 500, 777], [3, 17, 1], 2, dqk, dv, 0.6, dtype, 11))
    runs = [_bwd(N, dqk**-0.5, do, q, k, v, off, nt) for _ in range(2)]
    torch.cuda.synchronize()
    for name, a, b in zip(("dq", "dk", "dv"), *runs):
        assert torch.isfinite(a).all(), f"{name}: non-finite values"
        assert torch.equal(a.view(torch.int16), b.view(torch.int16)), f"{name}: two calls differ"
