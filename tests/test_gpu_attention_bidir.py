"""GPU: the non-causal (causal=False) attention against the fp64 oracle of the reference eager path's causal=False mask
(tests/bidir_oracle.py, pinned by tests/golden/bidir_attn_*.pt).

- The wgmma kernels (attn_*_bidir_wgmma_kernel, bf16 / fp16 at d = 32 / 64 / 128) and the generic kernels (every dtype
  and head dim, fp32, d = 256 and dqk < dv among them), forward and backward, under the mask options of
  test_gpu_attention_mixed_dims.MASK_OPTS, at lengths around the tile sizes and past max_seq_len, across the score scales
  of test_gpu_attention_numerics.SIGMAS, and on strided views of one uvqk buffer.  Every comparison is made on the whole
  tensor (assert_rel) and per 64-row segment (assert_rel_segments).
- Routing: hstu_attn_bidir_select_impl and the profiled kernel names.
- The backward is bitwise reproducible; torch.ops.hstu.hstu_mha(causal=False) and hstu_mha(causal=False) give the same
  results; a bf16 STULayer(causal=False) trains against the oracle stack; and the refusals.
"""
import ctypes as C

import pytest
import torch

import bidir_oracle as BO
from oracle import hstu_oracle as O
from test_gpu_attention import _random_case
from test_gpu_attention_deterministic import _kernels_of
from test_gpu_attention_mixed_dims import MASK_OPTS
from test_gpu_attention_numerics import SIGMAS, SWEEP, SWEEP_N, _compare
from util import assert_rel, normal_case, offsets_from

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda")
DIMS = [32, 64, 128]
DTYPES = [torch.bfloat16, torch.float16]
BIDIR_KERNELS = ("attn_fwd_bidir_wgmma_kernel", "attn_bwd_dkdv_bidir_wgmma_kernel", "attn_bwd_dq_bidir_wgmma_kernel")


def _lib():
    from generative_recommenders_b200 import _lib

    return _lib


def _run(impl, N, alpha, q, k, v, dout, off, nt, win=0, ctx=0, min_full=0, bwd=True):
    from generative_recommenders_b200.ops.hstu_attention import hstu_mha

    qd, kd, vd = (t.to(DEV).requires_grad_(bwd) for t in (q, k, v))
    out = hstu_mha(N, alpha, qd, kd, vd, off.to(DEV), causal=False, num_targets=None if nt is None else nt.to(DEV),
                   max_attn_len=win, contextual_seq_len=ctx, min_full_attn_seq_len=min_full, impl=impl)
    if not bwd:
        return out.detach(), None, None, None
    out.backward(dout.to(DEV))
    torch.cuda.synchronize()
    return out.detach(), qd.grad, kd.grad, vd.grad


def _oracle(N, alpha, q, k, v, dout, off, nt, win=0, ctx=0, min_full=0, bwd=True):
    off, nt = off.long(), None if nt is None else nt.long()
    kw = dict(num_targets=nt, max_attn_len=win, contextual_seq_len=ctx, min_full_attn_seq_len=min_full)
    out = BO.hstu_mha_fwd_bidir(N, alpha, q, k, v, off, **kw)
    return (out,) + (BO.hstu_mha_bwd_bidir(N, alpha, dout, q, k, v, off, **kw) if bwd else (None, None, None))


def _select(N, alpha, q, k, v, off, nt, win=0, ctx=0, min_full=0, impl=None, bwd=0):
    from generative_recommenders_b200.ops.hstu_attention import _fill_common

    L = _lib()
    qd, kd, vd, offd = q.to(DEV), k.to(DEV), v.to(DEV), off.to(DEV)
    p = L.AttnParams()
    _fill_common(p, N, alpha, qd, kd, vd, offd, None if nt is None else nt.to(DEV), win, ctx, min_full,
                 L.IMPL_AUTO if impl is None else impl)
    out = torch.empty(q.shape[0], q.shape[1], v.shape[2], dtype=v.dtype, device=DEV)
    p.out, p.o_row_stride, p.o_head_stride = out.data_ptr(), out.stride(0), out.stride(1)
    if bwd:
        p.dout = p.dq = p.dk = p.dv_out = out.data_ptr()
        p.do_row_stride = p.dq_row_stride = p.dk_row_stride = p.dv_row_stride = out.stride(0)
        p.do_head_stride = p.dq_head_stride = p.dk_head_stride = p.dv_head_stride = out.stride(1)
    return L.lib().hstu_attn_bidir_select_impl(C.byref(p), bwd)


def _case_args(c):
    return (c["max_seq_len"], c["alpha"], c["q"], c["k"], c["v"], c["dout"], c["seq_offsets"], c["num_targets"],
            c["max_attn_len"], c["contextual_seq_len"], c["min_full_attn_seq_len"])


@pytest.mark.parametrize("opts", MASK_OPTS)
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("d", DIMS)
def test_wgmma_vs_oracle_mask_options(d, dtype, opts):
    """Plain, targets, a window with min_full_attn_seq_len and a contextual prefix, a contextual prefix alone, int32."""
    targets, window, ctx, min_full, i32 = opts
    c = _random_case(7 * d + ctx + 3 * int(window), dtype, 4, 2, 260, 24, d, d, targets, window, ctx, min_full, i32=i32)
    args = _case_args(c)
    assert _select(*args[:5], args[6], args[7], *args[8:]) == _lib().IMPL_UMMA
    got = _run(_lib().IMPL_UMMA, *args)
    _compare(got, _oracle(*args), c["seq_offsets"], c["max_seq_len"], f"bidir wgmma d={d} {dtype} {opts}")


GENERIC_SHAPES = [(32, 32, torch.bfloat16), (64, 64, torch.float16), (128, 128, torch.bfloat16), (64, 64, torch.float32),
                  (256, 256, torch.bfloat16), (32, 64, torch.float16), (64, 128, torch.bfloat16), (25, 50, torch.float32)]


@pytest.mark.parametrize("opts", [MASK_OPTS[0], MASK_OPTS[2], MASK_OPTS[3]])
@pytest.mark.parametrize("dqk,dv,dtype", GENERIC_SHAPES)
def test_generic_vs_oracle(dqk, dv, dtype, opts):
    """The generic kernels at the wgmma dims (IMPL_GENERIC) and at every shape only they take (fp32, d = 256, dqk < dv,
    odd dims), where AUTO routes to them."""
    targets, window, ctx, min_full, i32 = opts
    c = _random_case(5 * dqk + dv + ctx, dtype, 3, 2, 200, 16, dqk, dv, targets, window, ctx, min_full, i32=i32)
    args = _case_args(c)
    wgmma = dtype != torch.float32 and dqk == dv and dqk <= 128
    if not wgmma:
        assert _select(*args[:5], args[6], args[7], *args[8:]) == _lib().IMPL_GENERIC
        assert _select(*args[:5], args[6], args[7], *args[8:], impl=_lib().IMPL_UMMA) == -2
    got = _run(_lib().IMPL_GENERIC if wgmma else _lib().IMPL_AUTO, *args)
    _compare(got, _oracle(*args), c["seq_offsets"], c["max_seq_len"], f"bidir generic ({dqk}, {dv}) {dtype} {opts}")


@pytest.mark.parametrize("dtype,i32", [(torch.bfloat16, True), (torch.float16, False)])
@pytest.mark.parametrize("d", DIMS)
def test_lengths_around_tiles_and_rows_past_max_seq_len(d, dtype, i32):
    """Lengths 0, 1, 63, 64, 65, 127, 128, 129, one of max_seq_len and one past it, whose rows past max_seq_len must be exact
    zeros in out, dq, dk and dv (the gradient buffers come from an allocator filled with NaN first)."""
    lengths, targets, N = [640, 0, 1, 63, 64, 65, 127, 128, 129, 700], [9, 0, 1, 3, 0, 5, 1, 2, 7, 4], 640
    q, k, v, do, off, nt = normal_case(lengths, targets, 2, d, 0.8, dtype, 99 + d, i32=i32)
    poison = torch.full((64 << 20,), float("nan"), device=DEV)
    del poison
    got = _run(_lib().IMPL_AUTO, N, d**-0.5, q, k, v, do, off, nt)
    _compare(got, _oracle(N, d**-0.5, q, k, v, do, off, nt), off, N, f"bidir lengths d={d} {dtype}")
    last = slice(int(off[-2]) + N, int(off[-1]))
    for name, a in zip(("out", "dq", "dk", "dv"), got):
        assert torch.equal(a[last].float().cpu(), torch.zeros_like(a[last].float().cpu())), f"{name}: rows past max_seq_len"


@pytest.mark.parametrize("sigma", SIGMAS)
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("d", DIMS)
def test_wgmma_across_score_scales(sigma, d, dtype):
    """q, k ~ N(0, sigma^2): rms(alpha S) from 0.09 to 4, where the tanh and the 1 + g2 cancellation of the backward show."""
    q, k, v, dout, off, nt = normal_case(SWEEP["lengths"], SWEEP["targets"], SWEEP["H"], d, sigma, dtype, 4049 + d)
    got = _run(_lib().IMPL_UMMA, SWEEP_N, d**-0.5, q, k, v, dout, off, nt)
    _compare(got, _oracle(SWEEP_N, d**-0.5, q, k, v, dout, off, nt), off, SWEEP_N, f"bidir d={d} {dtype} sigma={sigma}")


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("d", DIMS)
def test_long_sequence_window_context_and_targets(d, dtype):
    """Windowed key tiles well inside a 2048-row sequence (both range ends bounded), a contextual prefix, a full-attention
    tail and targets, at a large score scale."""
    N, win, ctx, min_full = 2048, 300, 70, 128
    q, k, v, dout, off, nt = normal_case([2048, 1100, 257, 64], [16, 3, 0, 2], 2, d, 1.5, dtype, 808 + d, i32=d == 64)
    got = _run(_lib().IMPL_UMMA, N, d**-0.5, q, k, v, dout, off, nt, win, ctx, min_full)
    _compare(got, _oracle(N, d**-0.5, q, k, v, dout, off, nt, win, ctx, min_full), off, N, f"bidir long d={d} {dtype}")


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("d", DIMS)
def test_strided_views_of_one_uvqk_buffer(d, dtype):
    """q, k, v as column views of one [L, H * (2 dv + 2 dqk)] buffer and the gradients written into views of another: the
    same bits as on contiguous tensors."""
    from generative_recommenders_b200.ops.hstu_attention import cuda_hstu_attention_bwd, cuda_hstu_attention_fwd

    H, N = 2, 300
    q, k, v, dout, off, nt = normal_case([300, 129, 64, 1], [5, 2, 0, 1], H, d, 1.0, dtype, 31 + d)
    L = q.shape[0]
    uvqk = torch.empty(L, 4 * H * d, dtype=dtype, device=DEV)
    _, vv, qq, kk = (t.view(L, H, d) for t in torch.split(uvqk, [H * d] * 4, dim=1))
    qq.copy_(q), kk.copy_(k), vv.copy_(v)
    offd, ntd, dod = off.to(DEV), nt.to(DEV), dout.to(DEV)
    alpha = d**-0.5
    out = cuda_hstu_attention_fwd(N, alpha, qq, kk, vv, offd, ntd, causal=False)
    duvqk = torch.empty_like(uvqk)
    _, dv_, dq_, dk_ = (t.view(L, H, d) for t in torch.split(duvqk, [H * d] * 4, dim=1))
    cuda_hstu_attention_bwd(N, alpha, dod, qq, kk, vv, dq_, dk_, dv_, offd, ntd, causal=False)
    qc, kc, vc = (t.to(DEV) for t in (q, k, v))
    out_c = cuda_hstu_attention_fwd(N, alpha, qc, kc, vc, offd, ntd, causal=False)
    g = [torch.empty_like(t) for t in (qc, kc, vc)]
    cuda_hstu_attention_bwd(N, alpha, dod, qc, kc, vc, *g, offd, ntd, causal=False)
    torch.cuda.synchronize()
    for name, a, b in (("out", out, out_c), ("dq", dq_, g[0]), ("dk", dk_, g[1]), ("dv", dv_, g[2])):
        assert torch.equal(a, b), name
    _compare((out, dq_, dk_, dv_), _oracle(N, alpha, q, k, v, dout, off, nt), off, N, f"bidir uvqk views d={d} {dtype}")


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("d", DIMS)
def test_routing_and_kernel_names(d, dtype):
    """AUTO selects the wgmma kernels forward and backward, and the profiler sees the bidir wgmma kernels run, not the
    generic ones and not the causal ones."""
    c = _random_case(11 + d, dtype, 3, 2, 300, 8, d, d, True, True, 3, 20)
    args = _case_args(c)
    sel = args[:5] + args[6:]
    assert _select(*sel) == _lib().IMPL_UMMA and _select(*sel, bwd=1) == _lib().IMPL_UMMA
    names = _kernels_of(lambda: _run(_lib().IMPL_AUTO, *args))
    for kname in BIDIR_KERNELS:
        assert any(kname in n for n in names), (kname, sorted(names))
    assert not any("generic" in n for n in names), sorted(names)
    for causal in ("attn_fwd_wgmma_kernel", "attn_bwd_dq_wgmma_kernel", "attn_bwd_dkdv_wgmma_kernel", "attn_bwd_wgmma_kernel"):
        assert not any(causal in n for n in names), sorted(names)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("d", DIMS + [256])
def test_backward_is_bitwise_reproducible(d, dtype):
    """No atomics on any path: two backward runs give the same bits (d = 256 runs the generic kernels)."""
    c = _random_case(3 + d, dtype, 4, 2, 400, 16, d, d, True, False, 0)
    args = _case_args(c)
    a = _run(_lib().IMPL_AUTO, *args)
    b = _run(_lib().IMPL_AUTO, *args)
    for name, x, y in zip(("out", "dq", "dk", "dv"), a, b):
        assert torch.equal(x, y), name


@pytest.mark.parametrize("dtype", DTYPES)
def test_torch_ops_and_hstu_mha_give_the_same_results(dtype):
    from generative_recommenders_b200 import torch_ops

    torch_ops.register()
    d = 32 if dtype == torch.bfloat16 else 64
    c = _random_case(21, dtype, 3, 2, 180, 8, d, d, True, True, 2, 0)
    args = _case_args(c)
    ref = _run(_lib().IMPL_AUTO, *args)
    N, alpha, q, k, v, dout, off, nt, win, ctx, mf = args
    qd, kd, vd = (t.to(DEV).requires_grad_() for t in (q, k, v))
    offd, ntd = off.to(DEV), nt.to(DEV)
    out = torch.ops.hstu.hstu_mha(N, alpha, qd, kd, vd, offd, False, ntd, None, win, mf, ctx, None, None, None, False, False, 0)
    out.backward(dout.to(DEV))
    for name, a, b in zip(("out", "dq", "dk", "dv"), (out.detach(), qd.grad, kd.grad, vd.grad), ref):
        assert torch.equal(a, b), f"hstu::hstu_mha {name}"
    o2 = torch.ops.hstu.hstu_mha_fwd(N, alpha, qd.detach(), kd.detach(), vd.detach(), offd, False, ntd, None, win, mf, ctx,
                                     None, None, None, 0)
    assert torch.equal(o2, ref[0])
    g = [torch.empty_like(t) for t in (qd, kd, vd)]
    torch.ops.hstu.hstu_mha_bwd(N, alpha, dout.to(DEV), qd.detach(), kd.detach(), vd.detach(), *g, offd, False, ntd, None,
                                win, mf, ctx, False, False, 0)
    for name, a, b in zip(("dq", "dk", "dv"), g, ref[1:]):
        assert torch.equal(a, b), f"hstu::hstu_mha_bwd {name}"


def test_stu_layer_non_causal_trains_against_the_oracle(monkeypatch):
    """A bf16 STULayer(causal=False) forward + backward (the fused block op on the wgmma kernels at d = 32) against the
    fp32 oracle stack under the non-causal mask, on the same bf16-valued parameters and inputs."""
    from generative_recommenders_b200.modules.stu import STULayer, STULayerConfig, STUStack

    torch.manual_seed(5)
    D, H, d = 64, 2, 32
    lengths, targets, N = [300, 77, 1, 190], [6, 2, 0, 9], 300
    stack = STUStack([STULayer(STULayerConfig(embedding_dim=D, num_heads=H, hidden_dim=d, attention_dim=d,
                                              output_dropout_ratio=0.0, causal=False, target_aware=True))])
    stack = stack.to(DEV).to(torch.bfloat16)
    off = offsets_from(lengths)
    nt = torch.tensor(targets)
    x = (torch.randn(int(off[-1]), D) * 0.5).to(torch.bfloat16)
    dout = torch.randn(int(off[-1]), D).to(torch.bfloat16)
    xd = x.to(DEV).requires_grad_()
    y = stack(x=xd, x_lengths=torch.tensor(lengths, device=DEV), x_offsets=off.to(DEV), max_seq_len=N, num_targets=nt.to(DEV))
    y.backward(dout.to(DEV))
    params = {n.split(".")[-1]: p.detach().float().cpu() for n, p in stack.named_parameters()}
    monkeypatch.setattr(O, "attn_valid_mask", BO.attn_valid_mask_bidir)  # the oracle stack under causal=False
    ry, rdx, rgrads = O.stu_stack_fwd_bwd(x.float(), off, N, nt, [params], H, d, d, dout)
    assert_rel(y, ry, "stu bidir y", tol=1.5e-2)
    assert_rel(xd.grad, rdx, "stu bidir dx", tol=3e-2)
    for n, p in stack.named_parameters():
        assert_rel(p.grad, rgrads[0][n.split(".")[-1]], f"stu bidir {n}", tol=3e-2)


def test_refusals():
    from generative_recommenders_b200.modules.stu import STULayer, STULayerConfig
    from generative_recommenders_b200.ops.hstu_attention import cuda_hstu_attention_fwd

    q = torch.randn(40, 1, 32, device=DEV, dtype=torch.bfloat16)
    off = torch.tensor([0, 40], device=DEV)
    with pytest.raises(RuntimeError, match="delta_q"):
        cuda_hstu_attention_fwd(40, 0.2, q[:8], q, q, off, delta_q_len=8, causal=False)
    with pytest.raises(RuntimeError, match="fp8"):
        f8 = q.to(torch.float8_e4m3fn)
        cuda_hstu_attention_fwd(40, 0.2, f8, f8, f8, off, causal=False)
    with pytest.raises(RuntimeError, match="relative bias"):
        cuda_hstu_attention_fwd(40, 0.2, q.float(), q.float(), q.float(), off, causal=False,
                                bias=(torch.zeros(79, device=DEV), None, None))
    layer = STULayer(STULayerConfig(embedding_dim=32, num_heads=1, hidden_dim=32, attention_dim=32, causal=False)).to(DEV)
    with pytest.raises(RuntimeError, match="causal"):
        layer.cached_forward(torch.randn(4, 32, device=DEV), None)
