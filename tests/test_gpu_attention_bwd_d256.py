"""The attention backward at head dim 256 on the wgmma kernels (bf16 and fp16).

With deterministic = 0, AUTO runs attn_bwd_dkdv_wgmma_kernel (two CTAs per key tile, one 128-column half of dK / dV each) and
attn_bwd_dq_wgmma_kernel (full-width dQ on 32-key tiles).  Checked here against the oracle in fp64, on the whole tensor
(assert_rel) and per 64-row segment (assert_rel_segments): which kernels run, the mask options of
test_attention_umma_vs_oracle with int32 and int64 offsets, lengths around the tile edges and a long sequence, the score-scale
sweep, extreme dO scales, rows past max_seq_len, sequence isolation, strided views of one uvqk / duvqk buffer, an STULayer
at attention_dim = hidden_dim = 256, agreement with the fp32 generic kernels at Lmax 4096, and bitwise repeatability (the
two kernels have no atomics).
"""
import ctypes as C

import pytest
import torch

from oracle import hstu_oracle as O
from test_gpu_attention import _random_case
from test_gpu_attention_deterministic import _assert_split_path, _bwd, _kernels_of, _params
from test_gpu_attention_numerics import (ISO_LENGTHS, ISO_N, ISO_TARGETS, SIGMAS, SWEEP_N, _check_isolated, _compare,
                                         _oracle, _poison, _run, _sweep_case)
from util import assert_rel, assert_rel_segments, normal_case, offsets_from

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda")
D = 256
DTYPES = [torch.bfloat16, torch.float16]


def _lib():
    from generative_recommenders_b200 import _lib

    return _lib


@pytest.mark.parametrize("dtype", DTYPES)
def test_d256_backward_runs_the_split_wgmma_kernels(dtype):
    _l = _lib()
    q, k, v, do, off, nt = (t.to(DEV) for t in normal_case([700, 300], [5, 2], 2, D, 0.5, dtype, 5))
    N, alpha = 768, D**-0.5
    lib = _l.lib()
    p = _params(N, alpha, q, k, v, off, False)
    assert lib.hstu_attn_select_impl(C.byref(p), 1) == _l.IMPL_UMMA
    assert lib.hstu_attn_workspace_bytes(C.byref(p), 1) == 0
    p.impl = _l.IMPL_UMMA
    assert lib.hstu_attn_select_impl(C.byref(p), 1) == _l.IMPL_UMMA
    # the deterministic flag keeps the generic kernels at d = 256
    p.deterministic, p.impl = 1, _l.IMPL_AUTO
    assert lib.hstu_attn_select_impl(C.byref(p), 1) == _l.IMPL_GENERIC
    _assert_split_path(_kernels_of(lambda: _bwd(N, alpha, do, q, k, v, off, nt)), f"d=256 {dtype}")
    names = _kernels_of(lambda: _run(_l.IMPL_UMMA, N, alpha, q, k, v, do, off, nt))
    _assert_split_path({n for n in names if "attn_bwd" in n or "convert" in n}, f"forced IMPL_UMMA d=256 {dtype}")


MASK_OPTS = [(False, False, 0, 0, False), (True, False, 0, 0, False), (True, True, 0, 0, False), (True, True, 7, 0, False),
             (True, True, 5, 33, False), (False, False, 4, 0, False), (True, False, 0, 0, True), (True, True, 5, 33, True)]


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("opts", MASK_OPTS)
def test_d256_mask_options_vs_oracle(dtype, opts):
    """The option sets of test_attention_umma_vs_oracle (targets, window, contextual prefix, min_full_attn_seq_len, int32
    offsets and targets) at d = 256."""
    _l = _lib()
    targets, window, ctx, min_full, i32 = opts
    c = _random_case(7256 + ctx, dtype, 5, 3, 300, 24, D, D, targets, window, ctx, min_full, i32=i32)
    args = (c["max_seq_len"], c["alpha"], c["q"], c["k"], c["v"], c["dout"], c["seq_offsets"], c["num_targets"],
            c["max_attn_len"], c["contextual_seq_len"], c["min_full_attn_seq_len"])
    got = _run(_l.IMPL_AUTO, *args)
    ref = _oracle(c["max_seq_len"], c["alpha"], c["q"], c["k"], c["v"], c["dout"], c["seq_offsets"].long(),
                  None if c["num_targets"] is None else c["num_targets"].long(), *args[8:])
    _compare(got, ref, c["seq_offsets"], c["max_seq_len"], f"d=256 {dtype} {opts}")


@pytest.mark.parametrize("dtype,i32", [(torch.bfloat16, True), (torch.float16, False)])
def test_d256_lengths_around_the_tiles_and_rows_past_max_seq_len(dtype, i32):
    """Lengths 0, 1, 63, 64, 65, 127, 128, 129, a 2048-row sequence at Lmax 2048, and one of 2100 rows whose rows past
    max_seq_len must come out as zeros (the gradient buffers start as NaN)."""
    lengths = [2048, 0, 1, 63, 64, 65, 127, 128, 129, 2100]
    targets = [9, 0, 1, 3, 0, 5, 1, 2, 7, 4]
    N, alpha = 2048, D**-0.5
    q, k, v, do, off, nt = normal_case(lengths, targets, 2, D, 0.8, dtype, 2560, i32=i32)
    got = _bwd(N, alpha, do.to(DEV), q.to(DEV), k.to(DEV), v.to(DEV), off.to(DEV), nt.to(DEV))
    torch.cuda.synchronize()
    ref = _oracle(N, alpha, q, k, v, do, off.long(), nt.long())[1:]
    for name, a, r in zip(("dq", "dk", "dv"), got, ref):
        assert_rel(a, r, f"d=256 lengths {dtype} {name}")
        assert_rel_segments(a, r, off, N, f"d=256 lengths {dtype} {name}")


@pytest.mark.parametrize("sigma", SIGMAS)
@pytest.mark.parametrize("dtype", DTYPES)
def test_d256_across_score_scales(sigma, dtype):
    """The sweep of test_wgmma_vs_oracle_across_score_scales, rms(alpha S) = 0.09 to 4, forward and backward."""
    q, k, v, dout, off, nt = _sweep_case(sigma, D, dtype)
    got = _run(_lib().IMPL_UMMA, SWEEP_N, D**-0.5, q, k, v, dout, off, nt)
    ref = _oracle(SWEEP_N, D**-0.5, q, k, v, dout, off, nt)
    _compare(got, ref, off, SWEEP_N, f"d=256 {dtype} rms(alpha S)={sigma**2:g}")


@pytest.mark.parametrize("dout_scale", [3e-8, 2e4])
def test_d256_is_invariant_to_the_scale_of_dout(dout_scale):
    """dS is a 16-bit tensor-core operand (a hi + lo pair of bf16): tiny and large output gradients keep the relative
    accuracy.  bf16 only: 3e-8 and 2e4 times N(0, 1) leave the range of fp16."""
    q, k, v, dout, off, nt = normal_case([700, 513, 64], [3, 9, 1], 3, D, 0.8, torch.bfloat16, 99)
    dout = (dout.float() * dout_scale).to(torch.bfloat16)
    N, alpha = 700, D**-0.5
    got = _bwd(N, alpha, dout.to(DEV), q.to(DEV), k.to(DEV), v.to(DEV), off.to(DEV), nt.to(DEV))
    torch.cuda.synchronize()
    ref = _oracle(N, alpha, q, k, v, dout, off, nt)[1:]
    for name, a, r in zip(("dq", "dk", "dv"), got, ref):
        assert_rel(a, r, f"dout x {dout_scale:g}: {name}")
        assert_rel_segments(a, r, off, N, f"dout x {dout_scale:g}: {name}")


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("value", ["nan", "inf"])
def test_d256_non_finite_rows_stay_in_their_sequence(dtype, value):
    """test_non_finite_rows_stay_in_their_sequence on the d = 256 backward: without atomics dq too is bitwise that of the run
    whose poisoned rows hold zeros."""
    q, k, v, dout, off, nt = normal_case(ISO_LENGTHS, ISO_TARGETS, 2, D, 0.7, dtype, 300 + D)
    alpha, impl = D**-0.5, _lib().IMPL_UMMA
    clean = [_poison(t, 0.0, 0) for t in (q, k, v, dout)]
    dirty = [_poison(t, value, i) for i, t in enumerate((q, k, v, dout))]
    got = _run(impl, ISO_N, alpha, *dirty, off, nt)
    base = _run(impl, ISO_N, alpha, *clean, off, nt)
    ref = _oracle(ISO_N, alpha, *clean, off, nt)
    _check_isolated(got, base, ref, f"d=256 {dtype} {value}")


@pytest.mark.parametrize("dtype", DTYPES)
def test_d256_strided_views_of_one_buffer(dtype):
    """q / k / v and dq / dk / dv as column slices of one [L, H * 4 d] uvqk / duvqk buffer, with targets, a window, a
    full-attention tail, a contextual prefix and int32 offsets; the first sequence runs past max_seq_len."""
    lengths, targets, N, win, min_full, ctx = [1100, 517, 300, 70], [9, 0, 4, 2], 1024, 150, 64, 37
    H, alpha = 2, D**-0.5
    q, k, v, do, off, nt = normal_case(lengths, targets, H, D, 1.0, dtype, 357, i32=True)
    L = q.shape[0]

    def views(buf):
        _, vv, qq, kk = torch.split(buf, [D * H] * 4, dim=1)
        return tuple(t.view(L, H, D) for t in (qq, kk, vv))

    uvqk = torch.empty(L, 4 * H * D, device=DEV, dtype=dtype)
    qd, kd, vd = views(uvqk)
    for dst, src in zip((qd, kd, vd), (q, k, v)):
        dst.copy_(src)
    duvqk = torch.full((L, 4 * H * D), float("nan"), device=DEV, dtype=dtype)
    grads = views(duvqk)
    got = _bwd(N, alpha, do.to(DEV), qd, kd, vd, off.to(DEV), nt.to(DEV), win, ctx, min_full, grads=grads)
    torch.cuda.synchronize()
    ref = _oracle(N, alpha, q, k, v, do, off.long(), nt.long(), win, ctx, min_full)[1:]
    for name, a, r in zip(("dq", "dk", "dv"), got, ref):
        assert_rel(a, r, f"strided d=256 {dtype} {name}")
        assert_rel_segments(a, r, off, N, f"strided d=256 {dtype} {name}")
    assert torch.isnan(duvqk[:, : D * H]).all(), "the u columns of duvqk were written"


def test_d256_stu_layer_vs_oracle():
    """An STULayer with attention_dim = hidden_dim = 256 (bf16, recompute on): its attention reads q / k / v from the strided
    uvqk and writes dq / dk / dv into the strided duvqk on the split wgmma kernels.  Forward, dx and every parameter gradient
    against the fp32 oracle, with the end-to-end budget of test_stu_stack_bf16_gradients_vs_oracle (1e-2: the GPU path stores
    bf16 activations between the ops of the layer, the oracle does not)."""
    from generative_recommenders_b200.modules.stu import STULayer, STULayerConfig, STUStack

    torch.manual_seed(23)
    Dm, H, N = 256, 2, 1024
    lengths, nts = [1024, 700, 129], [7, 2, 1]
    off = offsets_from(lengths)
    L = int(off[-1])
    stack = STUStack([STULayer(STULayerConfig(embedding_dim=Dm, num_heads=H, hidden_dim=D, attention_dim=D,
                                              output_dropout_ratio=0.0, target_aware=True))])
    with torch.no_grad():
        for n, p in stack.named_parameters():
            if "norm_weight" in n:
                p.add_(0.1 * torch.randn_like(p))
            if "norm_bias" in n or "beta" in n:
                p.add_(0.05 * torch.randn_like(p))
    stack = stack.to(DEV).to(torch.bfloat16)
    x = torch.randn(L, Dm).to(torch.bfloat16)
    dout = torch.randn(L, Dm).to(torch.bfloat16)
    xd = x.to(DEV).requires_grad_()
    out = {}

    def run():
        stack.zero_grad(set_to_none=True)
        xd.grad = None
        y = stack(x=xd, x_lengths=torch.tensor(lengths, device=DEV), x_offsets=off.to(DEV), max_seq_len=N,
                  num_targets=torch.tensor(nts, device=DEV))
        y.backward(dout.to(DEV))
        out["y"] = y

    names = _kernels_of(run)
    _assert_split_path({n for n in names if "attn_bwd" in n or "convert" in n}, "STULayer d=256")
    sd = {k: v.detach().float().cpu() for k, v in stack.state_dict().items()}
    params = [{k.split(".")[-1]: v for k, v in sd.items() if k.startswith("_stu_layers.0.")}]
    ry, rdx, rgrads = O.stu_stack_fwd_bwd(x.float(), off, N, torch.tensor(nts), params, H, D, D, dout.float())
    assert_rel(out["y"], ry, "STULayer d=256 y", tol=1e-2)
    assert_rel(xd.grad, rdx, "STULayer d=256 dx", tol=1e-2)
    for n, p in stack.named_parameters():
        assert_rel(p.grad, rgrads[0][n.split(".")[-1]], f"STULayer d=256 grad {n}", tol=1e-2)


def _grads(impl, N, alpha, q, k, v, do, off, nt):
    qq, kk, vv = (t.detach().clone().requires_grad_() for t in (q, k, v))
    from generative_recommenders_b200.common import HammerKernel
    from generative_recommenders_b200.ops.hstu_attention import hstu_mha

    hstu_mha(N, alpha, qq, kk, vv, off, num_targets=nt, kernel=HammerKernel.CUDA, impl=impl).backward(do)
    torch.cuda.synchronize()
    return qq.grad, kk.grad, vv.grad


@pytest.mark.parametrize("dtype", DTYPES)
def test_d256_matches_the_fp32_generic_kernels_at_lmax_4096(dtype):
    """At Lmax 4096, where the CPU oracle is too slow, the fp32 generic kernels on the same (rounded) values are the
    reference: they meet the oracle to 2e-5, so the bound is that of the oracle."""
    _l = _lib()
    lengths, targets, N = [4096, 3000, 2049], [11, 4, 1], 4096
    q, k, v, do, off, nt = (t.to(DEV) for t in normal_case(lengths, targets, 2, D, 0.8, dtype, 4096))
    alpha = D**-0.5
    got = _grads(_l.IMPL_AUTO, N, alpha, q, k, v, do, off, nt)
    ref = _grads(_l.IMPL_GENERIC, N, alpha, q.float(), k.float(), v.float(), do.float(), off, nt)
    for name, a, r in zip(("dq", "dk", "dv"), got, ref):
        assert_rel(a, r, f"d=256 vs fp32 generic {dtype} {name}")
        assert_rel_segments(a, r, off, N, f"d=256 vs fp32 generic {dtype} {name}")


@pytest.mark.parametrize("dtype", DTYPES)
def test_d256_backward_is_bitwise_repeatable(dtype):
    """No atomics in either kernel: every dq / dk / dv element is summed by one thread in a fixed order."""
    N = 4096
    q, k, v, do, off, nt = (t.to(DEV) for t in normal_case([N, N - 500, 777], [3, 17, 1], 2, D, 0.6, dtype, 11))
    runs = [_bwd(N, D**-0.5, do, q, k, v, off, nt) for _ in range(2)]
    torch.cuda.synchronize()
    for name, a, b in zip(("dq", "dk", "dv"), *runs):
        assert torch.isfinite(a).all(), f"{name}: non-finite values"
        assert torch.equal(a.view(torch.int16), b.view(torch.int16)), f"{name}: two calls differ"
